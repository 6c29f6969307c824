"""CPU oracle for the xclim per-grid-cell time-series hot path.  TEST INFRASTRUCTURE ONLY.

This module is a numpy restatement of the reference algorithms (Ouranosinc/xclim @ a8cbec8c,
v0.61.2-dev.7).  Every function cites the reference ``file:line`` it follows (paths relative to
``/root/reference/src/xclim``).  It is imported ONLY by ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs, as the checker -- never by the product
package ``xclim_b200`` (which fails loudly when the CUDA library is missing).

Pinning (see tests/test_oracle_golden.py, tests/golden/):
  * run-length cores and the Hyndman-Fan quantile are checked against the reference's OWN pure
    numpy/numba functions, executed in the authoring container by AST extraction from
    /root/reference (tests/golden/make_golden.py -> committed .npz fixtures), and against every
    synthetic known-answer value held by the reference's tests (SURVEY.md section 8c).
  * xarray-level semantics (resample grouping, rolling.construct padding, reindex by doy) cannot be
    executed here (xarray is absent); they are restated from the reference source and pinned only by
    the reference tests' known-answer values (test_calendar.py:83-103, test_indices.py:2354-2381,
    2594-2607 ...).
  * EQM (xsdba, a third-party dependency that is NOT under /root/reference; floor pin
    ``xsdba>=0.4.0``, pyproject.toml:111): **parity unpinned** -- restated from the published
    algorithm, anchored only on the reference call sites tests/test_xsdba.py:21-34,112-155.

Conventions: arrays are ``(time, ...)`` with time on axis 0 (the reference's ``dim="time"``);
``poff`` is the int array of P+1 period boundaries produced by ``resample(time=freq)`` (half-open
index ranges ``[poff[p], poff[p+1])``); ``doy``/``year`` are the ``time.dt.dayofyear`` / ``.year``
values.
"""
from __future__ import annotations

import operator

import numpy as np

# --------------------------------------------------------------------------------------------------
# a1  compare  (indices/generic.py:255-326)
# --------------------------------------------------------------------------------------------------
_BINARY_OPS = {">": "gt", "<": "lt", ">=": "ge", "<=": "le", "==": "eq", "!=": "ne"}


def get_op(op: str, constrain=None):
    """indices/generic.py:255-298 -- resolve an operator name, honouring ``constrain``."""
    if op in _BINARY_OPS:
        binary_op = _BINARY_OPS[op]
    elif op in _BINARY_OPS.values():
        binary_op = op
    else:
        raise ValueError(f"Operation `{op}` not recognized.")
    if constrain:
        allowed = []
        for c in ([constrain] if isinstance(constrain, str) else constrain):
            allowed.extend([c, _BINARY_OPS.get(c, c)])
        if op not in allowed:
            raise ValueError(f"Operation `{op}` not permitted for indice.")
    return getattr(operator, f"__{binary_op}__")


def compare(left, op, right, constrain=None):
    """indices/generic.py:301-326.  NaN compares False.  With numpy>=2 (NEP 50) a Python-float
    ``right`` is compared in ``left``'s dtype (float32); an array ``right`` promotes normally."""
    with np.errstate(invalid="ignore"):
        return get_op(op, constrain)(left, right)


# --------------------------------------------------------------------------------------------------
# resample helpers (xarray ``resample(time=freq)`` on a sorted daily axis == contiguous groups)
# --------------------------------------------------------------------------------------------------
def _groups(poff):
    poff = np.asarray(poff)
    return [(int(poff[p]), int(poff[p + 1])) for p in range(len(poff) - 1)]


def resample_reduce(x, poff, op):
    """``da.resample(time=freq).<op>(dim="time")`` (indices/generic.py:114).  xarray reductions skip
    NaN by default for float data; an all-NaN (or empty) group gives NaN for mean/min/max/std/var
    and 0 for sum."""
    x = np.asarray(x)
    outs = []
    for s, e in _groups(poff):
        blk = x[s:e]
        with np.errstate(all="ignore"), _quiet():
            if op == "sum":
                outs.append(np.nansum(blk, axis=0))
            elif op == "count":
                outs.append(np.sum(~np.isnan(blk), axis=0))
            else:
                outs.append(getattr(np, "nan" + op)(blk, axis=0))
    return np.stack(outs, axis=0)


class _quiet:
    def __enter__(self):
        import warnings
        self._cm = warnings.catch_warnings()
        self._cm.__enter__()
        warnings.simplefilter("ignore")

    def __exit__(self, *a):
        return self._cm.__exit__(*a)


# --------------------------------------------------------------------------------------------------
# a2  threshold_count (indices/generic.py:329-361)
# --------------------------------------------------------------------------------------------------
def threshold_count(x, op, threshold, poff, constrain=None):
    """indices/generic.py:357-361: ``(compare(da, op, thr) * 1).resample(time=freq).sum("time")``."""
    if constrain is None:
        constrain = (">", "<", ">=", "<=")
    c = compare(x, op, threshold, constrain) * 1
    return np.stack([c[s:e].sum(axis=0) for s, e in _groups(poff)], axis=0).astype(np.int64)


# --------------------------------------------------------------------------------------------------
# a19 MissingAny (core/missing.py:296-298, 318-322; applied core/indicator.py:1536-1547)
# --------------------------------------------------------------------------------------------------
def missing_any(x, poff, expected=None):
    """core/missing.py:310-322: True where a period has fewer valid (non-NaN) steps than ``expected``
    (``expected_count``, :64-160: the length of the complete period in the calendar; the observed
    number of steps when not given, which is the same for periods the series covers completely)."""
    valid = ~np.isnan(x)
    out = []
    for p, (s, e) in enumerate(_groups(poff)):
        out.append(valid[s:e].sum(axis=0) != ((e - s) if expected is None else int(expected[p])))
    return np.stack(out, axis=0)


# --------------------------------------------------------------------------------------------------
# a8  _cumsum_reset (indices/run_length.py:135-219)
# --------------------------------------------------------------------------------------------------
def _smallest_uint(n):
    """indices/run_length.py:135-139."""
    for dtype in (np.uint8, np.uint16, np.uint32, np.uint64):
        if np.iinfo(dtype).max > n:
            return dtype
    return np.uint64


def cumsum_reset(arr, index="last"):
    """Reset-on-zero cumulative sum along axis 0 (``100110111 -> 100120123``).

    Follows the fast track of indices/run_length.py:203-216: NaN -> 0 (``fillna``, :208) then the
    in-place scan ``arr[i] *= arr[i -/+ 1] + one`` of ``_cumsum_reset_np`` (:143-151).  The dtype is
    kept (bool inputs are promoted to the smallest uint holding T by ``fillna(typ(0))`` /
    ``*= ... + typ(1)``; float inputs stay float).
    """
    a = np.asarray(arr)
    n = a.shape[0]
    typ = _smallest_uint(n)
    if a.dtype == bool:
        a = a.astype(typ)
    else:
        a = np.where(np.isnan(a), 0, a).astype(a.dtype) if a.dtype.kind == "f" else a.copy()
    a = a.copy()
    one = a.dtype.type(1)
    if index == "last":
        for i in range(1, n):
            a[i] *= a[i - 1] + one
    else:
        for i in range(n - 2, -1, -1):
            a[i] *= a[i + 1] + one
    return a


def cumsum_reset_float(arr, index="last"):
    """``_cumsum_reset_xr(..., reset_on_zero=True)`` (indices/run_length.py:154-169): cumulative sum
    of the VALUES of each run of non-zero entries (used for float inputs by windowed_max_run_sum)."""
    a = np.asarray(arr, dtype=np.float64 if np.asarray(arr).dtype != np.float32 else np.float32)
    if index == "first":
        a = a[::-1]
    cs = np.cumsum(a, axis=0)
    cond = a == 0
    cs2 = np.where(cond, cs, np.nan)
    cs2[0] = 0
    # ffill along axis 0
    out = cs2.copy()
    for i in range(1, out.shape[0]):
        out[i] = np.where(np.isnan(out[i]), out[i - 1], out[i])
    res = cs - out
    if index == "first":
        res = res[::-1]
    return res


# --------------------------------------------------------------------------------------------------
# a9  rle (indices/run_length.py:223-272)
# --------------------------------------------------------------------------------------------------
def _shift(a, k, fill):
    """xarray ``shift({dim: k}, fill_value=fill)`` along axis 0."""
    out = np.full_like(a, fill)
    if k > 0:
        out[k:] = a[:-k]
    elif k < 0:
        out[:k] = a[-k:]
    else:
        out[...] = a
    return out


def rle(da, index="first"):
    """Whole-array run length (NOT an encoder): run length on the first (last) element of each run,
    NaN inside runs, 0 where the input is <= 0.  indices/run_length.py:254-272 step by step."""
    da = np.asarray(da)
    if index == "first":                                   # :255-256
        da = da[::-1]
    cs_s = cumsum_reset(da, "last").astype(np.float64)     # :259 (index="last" default of _cumsum_reset)
    daf = da.astype(np.float64)
    with np.errstate(invalid="ignore"):
        keep = _shift(daf, -1, 0) == 0                     # :264  da.shift(dim=-1, fill_value=0) == 0
        cs_s = np.where(keep, cs_s, np.nan)
        out = np.where(daf > 0, cs_s, 0)                   # :265
    if index == "first":                                   # :269-270
        out = out[::-1]
    return out


# --------------------------------------------------------------------------------------------------
# a10 rle_statistics / longest_run (indices/run_length.py:275-378)
# --------------------------------------------------------------------------------------------------
def _get_rl_stat(d, window, reducer):
    """indices/run_length.py:320-327.  ``reducer`` may also be a float q in [0, 1]: the quantile q, as "qNN" is
    the quantile 0.NN."""
    with np.errstate(all="ignore"), _quiet():
        dm = np.where(d >= window, d, np.nan)
        if isinstance(reducer, float):
            stat = np.nanquantile(dm, reducer, axis=0)
        elif reducer.startswith("q") and reducer[1:].isdigit():
            stat = np.nanquantile(dm, float(f"0.{reducer[1:]}"), axis=0)
        elif reducer == "count":
            stat = np.sum(~np.isnan(dm), axis=0).astype(np.float64)
        elif reducer == "sum":
            stat = np.nansum(dm, axis=0)
        else:
            stat = getattr(np, "nan" + reducer)(dm, axis=0)
        none = (np.isnan(d) | (d < window)).all(axis=0)
    return np.where(none, 0, stat)


def rle_statistics(da, reducer, window, poff=None, index="first"):
    """indices/run_length.py:275-335, general (non-ufunc) path.  ``poff`` is the *resample-after*
    frequency (runs attributed to the period holding their first element)."""
    d = rle(da, index=index)
    if poff is None:
        return _get_rl_stat(d, window, reducer)
    return np.stack([_get_rl_stat(d[s:e], window, reducer) for s, e in _groups(poff)], axis=0)


def longest_run(da, poff=None, index="first"):
    """indices/run_length.py:338-378."""
    return rle_statistics(da, "max", 1, poff=poff, index=index)


def resample_and_rl(da, resample_before_rl, compute, *args, poff, **kwargs):
    """indices/run_length.py:87-132 (+ helpers.py:937-943 non-dask branch)."""
    if resample_before_rl:
        return np.stack([compute(da[s:e], *args, **kwargs) for s, e in _groups(poff)], axis=0)
    return compute(da, *args, poff=poff, **kwargs)


# --------------------------------------------------------------------------------------------------
# a11 windowed_run_events / _count / _max_run_sum (indices/run_length.py:381-540)
# --------------------------------------------------------------------------------------------------
def _resample_sum(d, poff, fn=np.sum):
    if poff is None:
        return fn(d, axis=0)
    return np.stack([fn(d[s:e], axis=0) for s, e in _groups(poff)], axis=0)


def windowed_run_events(da, window, poff=None, index="first"):
    """indices/run_length.py:419-434 (general path)."""
    da = np.asarray(da)
    if window == 1:
        shift = 1 if index == "first" else -1
        daf = da.astype(np.float64)
        d = np.where(_shift(daf, shift, 0) == 0, 1, 0)
        d = np.where(daf == 1, d, 0)
    else:
        d = rle(da, index=index)
        with np.errstate(invalid="ignore"):
            d = np.where(d >= window, 1, 0)
    return _resample_sum(d, poff)


def windowed_run_count(da, window, poff=None, index="first"):
    """indices/run_length.py:473-488 (general path)."""
    da = np.asarray(da)
    if window == 1 and poff is None:
        return np.nansum(da.astype(np.float64), axis=0)
    d = rle(da, index=index)
    with np.errstate(invalid="ignore"):
        d = np.where(d >= window, d, 0)
    return _resample_sum(d, poff)


def windowed_max_run_sum(da, window, poff=None, index="first"):
    """indices/run_length.py:522-540."""
    da = np.asarray(da)
    d_rse = cumsum_reset_float(da, index=index)
    if window == 1 and poff is None:
        return d_rse.max(axis=0)
    d_rle = rle(da > 0, index=index)
    with np.errstate(invalid="ignore"):
        d = np.where(d_rle >= window, d_rse, 0)
    return _resample_sum(d, poff, np.max)


# --------------------------------------------------------------------------------------------------
# a12 first_run / last_run (indices/run_length.py:543-740), index outputs only (coord=False)
# --------------------------------------------------------------------------------------------------
def _find_boundary_run(runs, position):
    """indices/run_length.py:596-608."""
    n = runs.shape[0]
    if position == "last":
        runs = runs[::-1]
    dmax = runs.argmax(axis=0).astype(np.float64)
    out = np.where(dmax != runs.argmin(axis=0), dmax, np.nan)
    if position == "last":
        out = n - out - 1
    return out


def boundary_run(da, window, position, poff=None):
    """indices/run_length.py:610-640, general (non-ufunc) branches."""
    da = np.asarray(da)
    daf = np.where(np.isnan(da.astype(np.float64)), 0, da.astype(np.float64))  # :612
    if window == 1:
        d = daf
    else:
        d = cumsum_reset(daf, index=position)                                    # :632
        d = np.where(d >= window, 1, 0)                                          # :633
    if poff is None:
        return _find_boundary_run(d, position)
    return np.stack([_find_boundary_run(d[s:e], position) for s, e in _groups(poff)], axis=0)


def first_run(da, window, poff=None):
    return boundary_run(da, window, "first", poff)


def last_run(da, window, poff=None):
    return boundary_run(da, window, "last", poff)


# --------------------------------------------------------------------------------------------------
# a5/a6  spell_mask / spell_length_statistics (indices/generic.py:434-686)
# --------------------------------------------------------------------------------------------------
def _rolling(x, window, reducer):
    """``da.rolling(time=window).<reducer>()``: right-aligned, min_periods=window, NaN propagates."""
    T = x.shape[0]
    out = np.full(x.shape, np.nan, dtype=np.result_type(x.dtype, np.float32))
    fn = {"min": np.min, "max": np.max, "sum": np.sum, "mean": np.mean}[reducer]
    for t in range(window - 1, T):
        out[t] = fn(x[t - window + 1: t + 1], axis=0)
    return out


def spell_mask(data, window, win_reducer, op, thresh, min_gap=1):
    """indices/generic.py:499-540 (single variable, no weights)."""
    data = np.asarray(data)
    if window == 1:                                                             # :499-502
        is_in_spell = compare(data, op, thresh)
    elif (win_reducer == "min" and op in [">", ">=", "ge", "gt"]) or (
        win_reducer == "max" and op in ["`<", "<=", "le", "lt"]                  # sic (:504)
    ):
        mask = compare(data, op, thresh)                                         # :508
        cs_s = cumsum_reset(mask).astype(np.float64)                             # :514
        mf = mask.astype(np.float64)
        cs_s = np.where(_shift(mf, -1, 0) == 0, cs_s, np.nan)                    # :516
        with np.errstate(invalid="ignore"):
            v = np.where(cs_s >= window, cs_s, np.nan)
            v = np.where(mf > 0, v, 0)                                           # :518 stopper
        # bfill along time
        for t in range(v.shape[0] - 2, -1, -1):
            v[t] = np.where(np.isnan(v[t]), v[t + 1], v[t])
        with np.errstate(invalid="ignore"):
            is_in_spell = v > 0
    else:                                                                        # :519-535
        T = data.shape[0]
        pad = np.full((window,) + data.shape[1:], np.nan, dtype=np.result_type(data.dtype, np.float32))
        data_pad = np.concatenate([data.astype(pad.dtype), pad], axis=0)        # :520
        spell_value = _rolling(data_pad, window, win_reducer)                    # :527
        mask = compare(spell_value, op, thresh)                                  # :529
        rs = _rolling(mask.astype(np.float64), window, "sum")
        with np.errstate(invalid="ignore"):
            iis = rs >= 1                                                        # :533
        iis = _shift(iis, -(window - 1), False)
        is_in_spell = iis[:T]                                                    # :535
    if min_gap > 1:                                                              # :537-538
        is_in_spell = runs_with_holes(is_in_spell, 1, ~is_in_spell, min_gap).astype(bool)
    return is_in_spell


def runs_with_holes(da_start, window_start, da_stop, window_stop):
    """indices/run_length.py:844-888: 1 from the first step of a run of >= window_start True in
    ``da_start`` until the first step of a run of >= window_stop True in ``da_stop``."""
    a = np.asarray(da_start).astype(bool)
    b = np.asarray(da_stop).astype(bool)
    start_runs = cumsum_reset(a, index="first")                                   # :881
    stop_runs = cumsum_reset(b, index="first")                                    # :882
    start_positions = np.where(start_runs >= window_start, 1.0, np.nan)           # :883
    stop_positions = np.where(stop_runs >= window_stop, 0.0, np.nan)              # :884
    runs = np.where(np.isnan(stop_positions), start_positions, stop_positions)    # combine_first (:887)
    for t in range(1, runs.shape[0]):                                             # ffill
        runs[t] = np.where(np.isnan(runs[t]), runs[t - 1], runs[t])
    return np.where(np.isnan(runs), 0.0, runs)                                    # fillna(0)


def spell_length_statistics(data, threshold, window, win_reducer, op, spell_reducer, poff,
                            min_gap=1, resample_before_rl=True):
    """indices/generic.py:543-585 (no indexer): mask -> float32 -> resample_and_rl(rle_statistics,
    window=1)."""
    iis = spell_mask(data, window, win_reducer, op, threshold, min_gap=min_gap).astype(np.float32)
    return resample_and_rl(iis, resample_before_rl, rle_statistics, poff=poff,
                           reducer=spell_reducer, window=1).astype(np.float32)


def maximum_consecutive_dry_days(pr, thresh, poff, op="<", resample_before_rl=True):
    """indices/_threshold.py:2927-2937: spell_length_statistics(pr, thresh, 1, None, op, "max")
    then to_agg_units(..., "count") (x1 for daily data, core/units.py:704-712)."""
    return spell_length_statistics(pr, thresh, 1, None, op, "max", poff,
                                   resample_before_rl=resample_before_rl)


# --------------------------------------------------------------------------------------------------
# a15 NaN-aware Hyndman-Fan quantile (core/utils.py:326-557)
# --------------------------------------------------------------------------------------------------
def nan_quantile(arr, quantiles, alpha=1.0, beta=1.0):
    """Quantiles along axis 0 of ``arr`` -> array ``(nq,) + arr.shape[1:]`` (float64 for float32
    input because the interpolation weight is float64).  Written from the definition in
    core/utils.py:370-395 (virtual index), 417-461 (neighbour indexes and clamps), 464-491 (lerp with
    the difference taken in the DATA dtype and the gamma>=0.5 branch), 524-554 (NaN handling)."""
    arr = np.array(arr)                                   # copy (core/utils.py:362-365)
    quantiles = np.atleast_1d(np.asarray(quantiles, dtype=np.float64))
    n_axis = arr.shape[0]
    rest = arr.shape[1:]
    if n_axis == 0:
        return np.full((quantiles.size,) + rest, np.nan)
    if n_axis == 1:
        return np.broadcast_to(arr[0], (quantiles.size,) + rest).copy()
    flat = arr.reshape(n_axis, -1)
    srt = np.sort(flat, axis=0)                           # NaN sorted last (:538)
    n_valid = (n_axis - np.isnan(flat).sum(axis=0)).astype(np.float64)
    out = np.empty((quantiles.size, flat.shape[1]), dtype=np.result_type(arr.dtype, np.float64))
    with np.errstate(all="ignore"), _quiet():
        vmax = np.nanmax(flat, axis=0)                    # :554 fallback
        for qi, q in enumerate(quantiles):
            n = np.where(n_valid < 2, np.nan, n_valid)    # :527-530
            vi = n * q + (alpha + q * (1 - alpha - beta)) - 1          # :395
            prev = np.floor(vi)
            nxt = prev + 1
            above = vi >= n - 1                                          # :441-445
            prev = np.where(above, -1, prev)
            nxt = np.where(above, -1, nxt)
            below = vi < 0                                               # :447-450
            prev = np.where(below, 0, prev)
            nxt = np.where(below, 0, nxt)
            isn = np.isnan(vi)                                           # :451-457
            prev = np.where(isn, -1, prev).astype(np.intp)
            nxt = np.where(isn, -1, nxt).astype(np.intp)
            cols = np.arange(flat.shape[1])
            left = srt[prev, cols]
            right = srt[nxt, cols]
            gamma = vi - prev                                            # :412-414 (float64)
            diff = np.subtract(right, left)                              # data dtype (:486)
            lerp = np.add(left, diff * gamma)                            # :487
            lerp2 = np.subtract(right, diff * (1 - gamma))               # :488
            res = np.where(gamma >= 0.5, lerp2, lerp)
            out[qi] = np.where(np.isnan(res), vmax, res)                 # :554
    return out.reshape((quantiles.size,) + rest)


def calc_perc(arr_last_axis, percentiles, alpha=1.0, beta=1.0):
    """core/utils.py:279-323 convention: sample on the LAST axis, percentiles axis appended last."""
    a = np.moveaxis(np.asarray(arr_last_axis), -1, 0)
    q = nan_quantile(a, np.asarray(percentiles, dtype=np.float64) / 100.0, alpha, beta)
    return np.moveaxis(q, 0, -1)


# --------------------------------------------------------------------------------------------------
# a14 percentile_doy (core/calendar.py:395-494) and a16 doy re-mapping (core/calendar.py:690-790)
# --------------------------------------------------------------------------------------------------
def rolling_construct_center(x, window):
    """``arr.rolling(min_periods=1, center=True, time=window).construct("window")``
    (core/calendar.py:448): for every t the ``window`` neighbours ``x[t - window//2 + k]``,
    k = 0..window-1, NaN outside the series.  -> shape (T, window, ...)."""
    T = x.shape[0]
    h = window // 2
    out = np.full((T, window) + x.shape[1:], np.nan, dtype=np.result_type(x.dtype, np.float32))
    for k in range(window):
        off = k - h
        lo, hi = max(0, -off), min(T, T - off)
        out[lo:hi, k] = x[lo + off: hi + off]
    return out


def percentile_doy(x, year, doy, window=5, per=10.0, alpha=1.0 / 3.0, beta=1.0 / 3.0):
    """core/calendar.py:448-485.  Returns ``(n_doy, n_per) + x.shape[1:]`` float64 where n_doy is
    max(doy) (after the 366 -> interpolation step when present)."""
    x = np.asarray(x)
    year = np.asarray(year)
    doy = np.asarray(doy)
    per = np.atleast_1d(np.asarray(per, dtype=np.float64))
    rr = rolling_construct_center(x, window)                                   # :448
    years = np.unique(year)
    ndoy = int(doy.max())
    ny = len(years)
    # unstack (year, dayofyear) then stack (year, window): core/calendar.py:450-458
    rrr = np.full((ndoy, ny * window) + x.shape[1:], np.nan, dtype=rr.dtype)
    yidx = np.searchsorted(years, year)
    for t in range(x.shape[0]):
        rrr[doy[t] - 1, yidx[t] * window:(yidx[t] + 1) * window] = rr[t]
    p = np.empty((ndoy, per.size) + x.shape[1:], dtype=np.float64)
    for d in range(ndoy):
        p[d] = nan_quantile(rrr[d], per / 100.0, alpha, beta)                  # :469-479
    if ndoy == 366:                                                            # :484-485
        p = interpolate_doy_calendar(p[:365], 366)
    return p


def interpolate_doy_calendar(source, doy_max, doy_min=1):
    """core/calendar.py:690-726: fill NaN along doy (linear, interior only), re-label the doys on
    ``linspace(doy_min, doy_max, n)`` and linearly interpolate onto ``doy_min..doy_max``."""
    src = np.array(source, dtype=np.float64)
    n = src.shape[0]
    flat = src.reshape(n, -1)
    xs = np.arange(n, dtype=np.float64)
    for c in range(flat.shape[1]):                          # interpolate_na(dim="dayofyear") (:717)
        col = flat[:, c]
        ok = ~np.isnan(col)
        if ok.any() and not ok.all():
            col[:] = np.where(ok, col, np.interp(xs, xs[ok], col[ok], left=np.nan, right=np.nan))
    coords = np.linspace(doy_min, doy_max, n)               # :720
    target = np.arange(doy_min, doy_max + 1, dtype=np.float64)
    out = np.empty((target.size, flat.shape[1]))
    for c in range(flat.shape[1]):
        out[:, c] = np.interp(target, coords, flat[:, c])   # :722 .interp(dayofyear=range(...))
    return out.reshape((target.size,) + src.shape[1:])


def adjust_doy_calendar(table, target_doy, cal_max_doy=None):
    """core/calendar.py:729-760: re-map a doy table onto the doy range of the target time axis.
    ``cal_max_doy`` is ``max_doy[get_calendar(target)]`` (366 standard, 365 noleap, 360 360_day);
    the table is returned untouched when its last doy equals it (:748-750, 758-759; the
    ``has_similar_doys`` test at :752-754 compares bound methods and is never true)."""
    max_t, min_t = int(np.max(target_doy)), int(np.min(target_doy))
    if cal_max_doy is None:
        cal_max_doy = max_t
    if table.shape[0] == cal_max_doy:
        return table
    return interpolate_doy_calendar(table, max_t, min_t)


def resample_doy(table, target_doy, cal_max_doy=None):
    """core/calendar.py:763-790: ``reindex(time=arr.time.dt.dayofyear)`` gather -> (T, ...).
    After ``_interpolate_doy_calendar`` the table is labelled ``min_t..max_t``."""
    adoy = adjust_doy_calendar(table, target_doy, cal_max_doy)
    first = 1 if adoy is table else int(np.min(target_doy))
    return adoy[np.asarray(target_doy) - first]


def doy_threshold_count(x, table, doy, poff, op=">", cal_max_doy=None):
    """indices/_multivariate.py:1583-1590 + generic.py:357-361: float64 compare against the
    per-doy table (``table`` is (n_doy, ...))."""
    thresh = resample_doy(table, doy, cal_max_doy)
    return threshold_count(x, op, thresh, poff, constrain=(">", ">=") if op in (">", ">=") else ("<", "<="))


# --------------------------------------------------------------------------------------------------
# a17 percentile bootstrap (core/bootstrapping.py:128-211, 235-282)
# --------------------------------------------------------------------------------------------------
def bootstrap_doy_count(x, year, doy, poff, base_years, window=5, per=90.0, alpha=1 / 3., beta=1 / 3.,
                        op=">", table=None, cal_max_doy=None, feb29_index=59):
    """Zhang-2005 bootstrap of a doy-percentile exceedance count.

    ``poff`` groups must nest inside calendar years (freq YS/MS/QS...).  ``base_years`` =
    (first, last) year of the climatology.  For periods of in-base year y the result is the mean
    over the other base years s of the count obtained with thresholds computed on the base series
    in which block y is replaced by block s (core/bootstrapping.py:182-203); other periods use the
    plain table (:205-207).  Blocks of unequal length follow :255-279 (365 <-> 366 through
    ``convert_calendar``: Feb 29, at ``feb29_index`` of a year starting on 1 January, is dropped or
    filled with NaN).
    Returns float64 ``(P, ...)``.
    """
    x = np.asarray(x)
    year = np.asarray(year)
    doy = np.asarray(doy)
    if cal_max_doy is None:   # max_doy[get_calendar(target)] (core/calendar.py:748-750): a property of
        cal_max_doy = int(doy.max())  # the calendar, not of the sub-period being indexed
    y0, y1 = base_years
    in_base = (year >= y0) & (year <= y1)
    xb, yb, db = x[in_base], year[in_base], doy[in_base]
    if in_base.all():
        raise KeyError("`bootstrap` is unnecessary when all years are overlapping")
    if not in_base.any():
        raise KeyError("`bootstrap` is unnecessary when no year overlap")
    if table is None:
        table = percentile_doy(xb, yb, db, window, per, alpha, beta)[:, 0]
    byears = np.unique(yb)
    out = []
    for s_, e_ in _groups(poff):
        y = int(year[s_])
        blk = x[s_:e_]
        dblk = doy[s_:e_]
        if y0 <= y <= y1:
            acc = []
            pos_y = np.nonzero(yb == y)[0]
            for s in byears:
                if s == y:
                    continue
                pos_s = np.nonzero(yb == s)[0]
                z = xb.copy()
                ly, ls = len(pos_y), len(pos_s)
                if ls < 360 and ls < ly:                                 # :257-260 block left untouched
                    pass
                elif ls == ly:                                           # :264-265
                    z[pos_y] = xb[pos_s]
                elif ly == 365 and ls == 366:                            # :266-267 convert_calendar("noleap")
                    z[pos_y] = np.delete(xb[pos_s], feb29_index, axis=0)  # drops Feb 29
                elif ly == 366 and ls == 365:                            # :268-269 convert_calendar("366_day",
                    z[pos_y] = np.insert(xb[pos_s], feb29_index, np.nan, axis=0)  # missing=NaN): NaN on Feb 29
                elif ly < 365 and ls >= ly:                              # :270-273
                    z[pos_y] = xb[pos_s][:ly]
                else:
                    raise NotImplementedError("unequal year blocks")
                tab = percentile_doy(z, yb, db, window, per, alpha, beta)[:, 0]
                acc.append(threshold_count(blk, op, resample_doy(tab, dblk, cal_max_doy), [0, e_ - s_])[0])
            out.append(np.mean(np.stack(acc, axis=0), axis=0))
        else:
            out.append(threshold_count(blk, op, resample_doy(table, dblk, cal_max_doy), [0, e_ - s_])[0].astype(np.float64))
    return np.stack(out, axis=0)


# --------------------------------------------------------------------------------------------------
# a3/a4  resample reductions, thresholded sums, rolling (indices/generic.py:83-174, 1514-1552)
# --------------------------------------------------------------------------------------------------
def select_resample_op(x, op, poff):
    """indices/generic.py:110-125 (no indexer)."""
    return resample_reduce(x, poff, op)


def cumulative_difference(x, threshold, op, poff):
    """indices/generic.py:1514-1552: ``(x - t).clip(0)`` for > / >=, ``(t - x).clip(0)`` for < / <=,
    then resample-sum."""
    x = np.asarray(x)
    if op in (">", ">=", "gt", "ge"):
        diff = np.clip(x - x.dtype.type(threshold), 0, None)
    else:
        diff = np.clip(x.dtype.type(threshold) - x, 0, None)
    return resample_reduce(diff, poff, "sum")


def rolling(x, window, op, center=False):
    """``da.rolling(time=window, center=center).<op>()`` (min_periods=window, NaN for incomplete or
    NaN-holding windows)."""
    x = np.asarray(x)
    r = _rolling(x, window, op)
    if center:
        r = _shift(r, -(window // 2), np.nan)
    return r


def select_rolling_resample_op(x, op, window, poff, window_center=True, window_op="mean"):
    """indices/generic.py:169-174."""
    return resample_reduce(rolling(x, window, window_op, center=window_center), poff, op)


def window_stat_rule(x, window, stat):
    """The kernels' window statistic (DESIGN §4, ``window_stat`` in csrc/rolling.cu), right-aligned: the value
    at t covers x[t-window+1 .. t] (NaN for t < window-1).  A sum is the float64 sum of the window's values
    from the oldest to the newest, one add at a time (np.sum would pair them up), rounded once to float32; a
    mean is (float)(sum / window); min and max are taken in float32.  A window holding a NaN is NaN."""
    x = np.asarray(x, dtype=np.float32)
    out = np.full(x.shape, np.nan, dtype=np.float32)
    n = x.shape[0] - window + 1
    if n <= 0:
        return out
    with np.errstate(all="ignore"):
        if stat in ("sum", "mean"):
            s = np.zeros((n,) + x.shape[1:], dtype=np.float64)
            for k in range(window):
                s = s + x[k:k + n].astype(np.float64)
            out[window - 1:] = (s / window if stat == "mean" else s).astype(np.float32)
        else:
            fn = np.fmin if stat == "min" else np.fmax
            m = x[:n].copy()
            nan = np.isnan(m)
            for k in range(1, window):
                m = fn(m, x[k:k + n])
                nan |= np.isnan(x[k:k + n])
            out[window - 1:] = np.where(nan, np.float32(np.nan), m)
    return out


def spell_mask_rule(x, window, stat, op, thresh):
    """The kernels' spell mask: step t is in a spell if some length-``window`` block that lies fully inside the
    series and contains t has (window statistic op float32(thresh)); a NaN window only satisfies ``!=``.
    The reference pads the series end with NaN instead (spell_mask above), which differs under ``!=`` only."""
    x = np.asarray(x, dtype=np.float32)
    T = x.shape[0]
    cond = np.zeros(x.shape, dtype=bool)           # cond[i]: block [i, i+window-1]
    with np.errstate(invalid="ignore"):
        cond[:T - window + 1] = compare(window_stat_rule(x, window, stat)[window - 1:], op, np.float32(thresh))
    mask = cond.copy()
    for k in range(1, window):
        mask[k:] |= cond[:T - k]
    return mask


def rolling_rule(x, window, stat, center=False):
    """``rolling(time=window, center=center).<stat>()`` under the kernels' window rule: the value labelled t
    covers the window ending at t + shift (shift = window // 2 when centred); incomplete windows are NaN."""
    r = window_stat_rule(x, window, stat)
    return _shift(r, -(window // 2), np.nan) if center else r


def period_stat_rule(vals, poff, stat):
    """Per-period statistic of float32 values as the kernels' StatAcc takes it: NaN skipped, sum and sum of
    squares in float64 in time order, rounded once; var = E[v^2] - E[v]^2 clamped at 0 (one pass).  The rule
    itself is oracle/stat_rule.py's period_stat."""
    from oracle import stat_rule
    return stat_rule.period_stat(vals, poff, stat)


def tg_mean(tas, poff):
    """indices/_simple.py:113."""
    return select_resample_op(tas, "mean", poff)


# --------------------------------------------------------------------------------------------------
# a20 Empirical quantile mapping (xsdba; PARITY UNPINNED -- see module docstring)
# --------------------------------------------------------------------------------------------------
def eqm_nodes(nquantiles):
    """xsdba.utils.equally_spaced_nodes(n, eps=None): ``linspace(1/2n, 1-1/2n, n)``."""
    dq = 1.0 / nquantiles / 2.0
    return np.linspace(dq, 1.0 - dq, nquantiles)


def eqm_train(ref, hist, nquantiles=20, kind="+"):
    """EmpiricalQuantileMapping.train(group="time"): NaN-aware linear (type 7) quantiles of ref and
    hist at the nodes; ``af = ref_q - hist_q`` ("+") or ``ref_q / hist_q`` ("*").  Results in the
    data dtype (float32 nodes, float32 outputs).  Returns (af, hist_q) each ``(nq, ...)``."""
    q = eqm_nodes(nquantiles).astype(ref.dtype)
    with _quiet():
        ref_q = np.nanquantile(np.asarray(ref, np.float64), q.astype(np.float64), axis=0).astype(ref.dtype)
        hist_q = np.nanquantile(np.asarray(hist, np.float64), q.astype(np.float64), axis=0).astype(hist.dtype)
    with np.errstate(all="ignore"):
        af = ref_q - hist_q if kind == "+" else ref_q / hist_q
    return af, hist_q


def eqm_adjust(sim, af, hist_q, kind="+", interp="linear"):
    """EmpiricalQuantileMapping.adjust(extrapolation="constant"): per element, interpolate ``af``
    over ``hist_q`` at ``sim`` (linear, or nearest with ties to the lower node), constant end
    factors outside ``[hist_q[0], hist_q[-1]]``, then apply additively / multiplicatively."""
    sim = np.asarray(sim)
    T = sim.shape[0]
    s2 = sim.reshape(T, -1)
    af2 = af.reshape(af.shape[0], -1)
    hq2 = hist_q.reshape(hist_q.shape[0], -1)
    out = np.full(s2.shape, np.nan, dtype=sim.dtype)
    for c in range(s2.shape[1]):
        xq, yq = hq2[:, c].astype(np.float64), af2[:, c].astype(np.float64)
        ok = ~(np.isnan(xq) | np.isnan(yq))
        sv = s2[:, c].astype(np.float64)
        m = ~np.isnan(sv)
        if not ok.any() or not m.any():
            continue
        xq, yq = xq[ok], yq[ok]
        if interp == "linear":
            f = np.interp(sv[m], xq, yq)
        else:
            # scipy.interpolate.interp1d(kind="nearest"): x_bds = x/2; x_bds[1:] + x_bds[:-1] evaluated in
            # the dtype of hist_q (float32), searchsorted(side="left") -> ties go to the lower node
            h32 = hq2[:, c][ok] / np.float32(2.0)
            bds = h32[1:] + h32[:-1]
            f = yq[np.searchsorted(bds, s2[:, c][m], side="left")]
        res = sv[m] + f if kind == "+" else sv[m] * f
        col = np.full(T, np.nan)
        col[m] = res
        out[:, c] = col.astype(sim.dtype)
    return out.reshape(sim.shape)


# --------------------------------------------------------------------------------------------------
# a12 (cont.) date-bounded runs and seasons, per GROUP (indices/run_length.py:891-1331).  ``da`` is a
# boolean group (n, ...); ``mid`` is the index of the MM-DD date inside the group (``index_of_date``,
# :1621-1665) or None when the date is absent / not requested.
# --------------------------------------------------------------------------------------------------
def _masked(da, keep):
    """``da.where(keep)``: NaN outside (later ``fillna(0)`` -> False, run_length.py:612)."""
    daf = np.asarray(da, dtype=np.float64)
    k = keep.reshape((-1,) + (1,) * (daf.ndim - 1))
    return np.where(k, daf, np.nan)


def first_run_after_date(da, window, mid):
    """indices/run_length.py:1204-1244."""
    da = np.asarray(da)
    if mid is None:
        return np.full(da.shape[1:], np.nan)
    idx = np.arange(da.shape[0])
    return boundary_run(_masked(da, idx >= mid), window, "first")


def last_run_before_date(da, window, mid):
    """indices/run_length.py:1247-1284."""
    da = np.asarray(da)
    if mid is None:
        return np.full(da.shape[1:], np.nan)
    idx = np.arange(da.shape[0])
    return boundary_run(_masked(da, idx <= mid), window, "last")


def first_run_before_date(da, window, mid, has_date=True):
    """indices/run_length.py:1287-1331 (``has_date=False``: ``date=None`` -> plain first_run)."""
    da = np.asarray(da)
    if has_date:
        if mid is None:
            return np.full(da.shape[1:], np.nan)
        idx = np.arange(da.shape[0])
        da = _masked(da, idx < mid + window - 1)
    return boundary_run(da, window, "first")


def run_end_after_date(da, window, mid):
    """indices/run_length.py:1148-1201 (index outputs)."""
    da = np.asarray(da).astype(bool)
    if mid is None:
        return np.full(da.shape[1:], np.nan)
    idx = np.arange(da.shape[0])
    end = boundary_run(_masked(~da, idx >= mid), window, "first")
    beg = boundary_run(_masked(da, idx < mid), window, "first")
    end = np.where(np.isnan(end) & ~np.isnan(beg), da.shape[0] - 1, end)
    return np.where(np.isnan(beg), np.nan, end)


def season_group(da, window, mid, has_date=True):
    """indices/run_length.py:998-1110 with ``coord=False``: (start, end, length) of one group."""
    da = np.asarray(da).astype(bool)
    n = da.shape[0]
    beg = first_run_before_date(da, window, mid, has_date)                       # season_start (:929)
    idx = np.arange(n).reshape((-1,) + (1,) * (da.ndim - 1))
    not_da = np.where(idx >= np.where(np.isnan(beg), 0, beg), (~da).astype(np.float64), np.nan)   # :977
    if has_date:
        end = first_run_after_date(not_da, window, mid)                          # :978
    else:
        end = boundary_run(not_da, window, "first")                              # date=None -> index 0
    length = np.where(np.isnan(beg), 0, np.where(np.isnan(end), n - beg, end - beg))   # :1072-1077
    end = np.where(np.isnan(end) & ~np.isnan(beg), n - 1, end)                   # :1081-1082
    end = np.where(np.isnan(beg), np.nan, end)
    return beg, end, length


def season(cond, window, mids, poff, stat, doy=None, has_date=True):
    """indices/generic.py:769-853 after the compare: per period ``season_*`` (start/end as dayofyear)."""
    outs = []
    for p, (s, e) in enumerate(_groups(poff)):
        beg, end, length = season_group(cond[s:e], window, mids[p] if has_date else None, has_date)
        if stat == "length":
            outs.append(length)
        else:
            v = beg if stat == "start" else end
            t = np.where(np.isnan(v), 0, v).astype(int) + s
            outs.append(np.where(np.isnan(v), np.nan, np.asarray(doy)[t]))
    return np.stack(outs, axis=0)


# --------------------------------------------------------------------------------------------------
# missing-value masks beyond "any" (core/missing.py:338-522)
# --------------------------------------------------------------------------------------------------
def missing_pct(x, poff, tolerance, expected=None):
    """core/missing.py:476-482 (``count`` = ``expected_count``, see :func:`missing_any`)."""
    valid = ~np.isnan(x)
    out = []
    for p, (s, e) in enumerate(_groups(poff)):
        n = (e - s) if expected is None else int(expected[p])
        out.append((n - valid[s:e].sum(axis=0)) / n >= tolerance)
    return np.stack(out)


def at_least_n_valid(x, poff, n):
    """core/missing.py:517-522."""
    valid = ~np.isnan(x)
    return np.stack([valid[s:e].sum(axis=0) < n for s, e in _groups(poff)])


def missing_wmo(x, poff_month, parent, n_parent, nm=11, nc=5, expected_month=None, months_per_period=None):
    """core/missing.py:434-450 at the monthly step (``count`` = days of the complete month when
    ``expected_month`` is given), then MissingAny over the months of every coarser period (:384-391:
    missing months are NaN, and a period holding fewer than ``months_per_period`` months is missing).
    ``parent[m]`` = index of the coarser period holding month m."""
    valid = ~np.isnan(x)
    miss_m = []
    for m, (s, e) in enumerate(_groups(poff_month)):
        n = (e - s) if expected_month is None else int(expected_month[m])
        missing_days = n - valid[s:e].sum(axis=0)
        longest = rle_statistics(~valid[s:e], "max", 1)
        miss_m.append((missing_days >= nm) | (longest >= nc))
    miss_m = np.stack(miss_m)
    out = np.zeros((n_parent,) + x.shape[1:], bool)
    for m, p in enumerate(parent):
        out[p] |= miss_m[m]
    if months_per_period is not None:
        short = np.bincount(np.asarray(parent), minlength=n_parent) != months_per_period
        out |= short.reshape((-1,) + (1,) * (x.ndim - 1))
    return out


def select_time_mask(month, day, doy, calendar, season=None, months=None, doy_bounds=None, date_bounds=None):
    """core/calendar.py:1259-1376 as a boolean step mask (inclusive bounds)."""
    month, day, doy = np.asarray(month), np.asarray(day), np.asarray(doy)
    if season is not None:
        names = {12: "DJF", 1: "DJF", 2: "DJF", 3: "MAM", 4: "MAM", 5: "MAM", 6: "JJA", 7: "JJA", 8: "JJA",
                 9: "SON", 10: "SON", 11: "SON"}
        want = [season] if isinstance(season, str) else season
        return np.array([names[int(m)] in want for m in month])
    if months is not None:
        return np.isin(month, months)
    if doy_bounds is not None:
        a, b = doy_bounds
        doys = np.arange(a, b + 1) if a <= b else np.concatenate((np.arange(a, 367), np.arange(0, b + 1)))
        return np.isin(doy, doys)
    # date bounds: day numbers in the (uniform) calendar, or all_leap numbering for standard calendars
    leap = calendar not in ("noleap", "365_day", "360_day")
    def num(m, d):
        if calendar == "360_day":
            return (m - 1) * 30 + d
        dpm = [31, 29 if leap else 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31]
        return sum(dpm[: m - 1]) + d
    cur = np.array([num(int(m), int(d)) for m, d in zip(month, day)])
    a, b = (num(*(int(v) for v in s.split("-"))) for s in date_bounds)
    doys = np.arange(a, b + 1) if a <= b else np.concatenate((np.arange(a, 367), np.arange(0, b + 1)))
    return np.isin(cur, doys)
