"""CUDA implementations behind the signatures of ``xclim.indices.generic``.

Each function keeps the reference's name, argument meaning and error behaviour (cited below) but
runs as ONE streaming CUDA kernel over the ``(time, lat, lon)`` float32 buffer.
"""
from __future__ import annotations

import numpy as np

from . import _lib, device
from .field import attrs_of, dims_of, is_xarray, raw_values, time_axis_of, wrap_like
from .options import OPTIONS
from .units import threshold_in_units_of, to_agg_units_attrs


# --------------------------------------------------------------------------------------- plumbing
def _unwrap(da, indexer=None):
    dims = dims_of(da)
    if "time" not in dims:
        raise ValueError("input must have a `time` dimension")
    tpos = dims.index("time")
    x2d, cell_shape = device.to_time_cell(raw_values(da), tpos)
    other = tuple(d for d in dims if d != "time")
    ta = time_axis_of(da)
    if indexer:  # select_time(da, **indexer), drop=False (core/calendar.py:1259-1376)
        keep = ta.select_mask(**indexer)
        if not keep.all():
            x2d = device.mask_steps(x2d, keep)
    return x2d, cell_shape, other, ta


def _period_time(da, ta, freq):
    """Time coordinate of the resampled output (period labels)."""
    labels = ta.period_labels(freq)
    if ta.coord is not None:  # xarray input: let xarray build the exact resampled index
        try:
            return ta.coord.resample(time=freq).first().time
        except Exception:  # pragma: no cover
            pass
    return np.array(labels)


def _wrap_periods(da, out2d, cell_shape, other_dims, ta, freq, attrs, dtype=None, name=None):
    """(P, C) device result -> container of the input's family with dims (time=periods, *space); with
    ``freq=None`` (reduction over the whole series) the time dimension is dropped, as the reference's
    ``.reduce(dim="time")`` does."""
    vals = out2d.reshape((out2d.shape[0],) + cell_shape)
    if freq is None:
        vals = vals[0]
    if OPTIONS["device_outputs"] and not is_xarray(da) and getattr(vals, "is_cuda", False):
        if dtype is not None:      # same dtype as the host path, converted where the data are
            import torch
            vals = vals.to(getattr(torch, np.dtype(dtype).name))
    else:
        vals = vals.cpu().numpy()
        if dtype is not None:
            vals = vals.astype(dtype, copy=False)
    if freq is None:
        return wrap_like(da, vals, tuple(other_dims), attrs=attrs, name=name)
    return wrap_like(da, vals, ("time",) + other_dims, time=_period_time(da, ta, freq), attrs=attrs, name=name)


def _scalar_threshold(threshold):
    """A Python number compares in float32 (numpy>=2 weak scalar); a 0-d float64 array/np.float64
    compares in float64 (indices/generic.py:301-326 + NEP 50).  np.float64 subclasses float, so it is tested
    first."""
    if isinstance(threshold, np.floating):
        return float(threshold), threshold.dtype == np.float64
    if isinstance(threshold, (int, float)):
        return float(threshold), False
    arr = np.asarray(getattr(threshold, "values", threshold))
    if arr.ndim == 0:
        return float(arr), arr.dtype == np.float64
    raise NotImplementedError("array thresholds are supported through the doy-percentile entry points only")


def _array_threshold(threshold, da, cell_shape, other_dims, x2d):
    """A threshold given as an array (labelled like the data, or a bare array of the data's shape / of its
    spatial shape) -> (float64 device tensor (T|1, C), varies_in_time); None for scalars."""
    import torch
    from .field import Field
    if isinstance(threshold, (int, float, str, np.floating, np.integer)):
        return None
    labelled = isinstance(threshold, Field) or is_xarray(threshold)
    vals = raw_values(threshold) if labelled else threshold
    if getattr(vals, "ndim", 0) == 0:
        return None
    if hasattr(vals, "is_cuda"):
        t = vals.to(x2d.device, torch.float64)
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(vals, dtype=np.float64))).to(x2d.device)
    T = x2d.shape[0]
    if labelled:
        tdims = dims_of(threshold)
        per_time = "time" in tdims
        want = (("time",) if per_time else ()) + tuple(other_dims)
        if set(tdims) != set(want):
            raise ValueError(f"threshold dims {tdims} do not match the data dims {('time',) + tuple(other_dims)}")
        t = t.permute([tdims.index(d) for d in want])
    else:
        per_time = tuple(t.shape) == (T,) + tuple(cell_shape)
        if not per_time and tuple(t.shape) != tuple(cell_shape):
            raise ValueError(f"threshold shape {tuple(t.shape)} matches neither the data nor its spatial shape")
    t = t.contiguous().reshape((T if per_time else 1), -1)
    return t, per_time


# --------------------------------------------------------------------------------- a1  get_op/compare
def get_op(op, constrain=None):
    """indices/generic.py:255-298: validate an operator name; returns its C-ABI code."""
    return _lib.op_code(op, constrain)


# --------------------------------------------------------------------------------- a2 threshold_count
def threshold_count(da, op, threshold, freq, constrain=None):
    """Count of steps where ``da op threshold`` per period -- indices/generic.py:329-361.

    Output: int64 ``(time=periods, ...)`` like ``(cond * 1).resample(time=freq).sum("time")``.
    """
    if constrain is None:
        constrain = (">", "<", ">=", "<=")
    code = get_op(op, constrain)
    x2d, cell_shape, other, ta = _unwrap(da)
    arr = _array_threshold(threshold, da, cell_shape, other, x2d)
    if arr is not None:      # DataArray / array threshold: compared in float64 (SURVEY.md A.1)
        out = device.period_count_arr(x2d, ta.period_offsets(freq), code, arr[0], arr[1])
    else:
        thr, f64 = _scalar_threshold(threshold)
        out, _ = device.period_count(x2d, ta.period_offsets(freq), code, thr, cmp_f64=f64)
    return _wrap_periods(da, out, cell_shape, other, ta, freq, attrs_of(da), dtype=np.int64)


def domain_count(da, low, high, freq):
    """Count of steps with ``low < da <= high`` per period -- indices/generic.py:364-392.
    NaN fails both comparisons, so for low <= high the count equals #(da > low) - #(da > high)."""
    x2d, cell_shape, other, ta = _unwrap(da)
    poff = ta.period_offsets(freq)
    low, high = float(low), float(high)
    a, _ = device.period_count(x2d, poff, _lib.OPS[">"], low)
    if low <= high:
        b, _ = device.period_count(x2d, poff, _lib.OPS[">"], high)
        a = a - b
    else:
        a = a * 0
    return _wrap_periods(da, a, cell_shape, other, ta, freq, attrs_of(da), dtype=np.int64)


# --------------------------------------------------------------------------------- a3 resample ops
def select_resample_op(da, op, freq="YS", out_units=None, **indexer):
    """Per-period reduction -- indices/generic.py:83-125 (string ops only)."""
    if not isinstance(op, str) or op not in _lib.STATS:
        raise NotImplementedError(f"resample op {op!r} is not supported by the xclim_b200 hot path")
    x2d, cell_shape, other, ta = _unwrap(da, indexer)
    out, _ = device.period_reduce(x2d, ta.period_offsets(freq), _lib.STATS[op])
    attrs = attrs_of(da)
    attrs.update({"units": out_units} if out_units is not None else to_agg_units_attrs(da, op.replace("integral", "sum")))
    dtype = np.int64 if op == "count" else None
    return _wrap_periods(da, out, cell_shape, other, ta, freq, attrs, dtype=dtype)


_MONTH_ABBREVIATIONS = {1: "JAN", 2: "FEB", 3: "MAR", 4: "APR", 5: "MAY", 6: "JUN", 7: "JUL", 8: "AUG", 9: "SEP",
                        10: "OCT", 11: "NOV", 12: "DEC"}


def default_freq(**indexer):
    """Default resampling frequency of an indexer -- indices/generic.py:224-252: "YS-JAN", or the year starting
    in the indexer's first month ("YS-DEC" for a season)."""
    freq = "YS-JAN"
    if indexer:
        group, value = indexer.popitem()
        if group == "season":
            month = 12      # the "season" scheme is based on YS-DEC
        elif group == "month":
            month = int(np.take(value, 0))
        elif group == "doy_bounds":
            # the month of day value[0] of 2004 (a leap year), as cftime.num2date(value[0] - 1, "days since
            # 2004-01-01") gives it
            month = int((np.datetime64("2004-01-01") + np.timedelta64(int(value[0]) - 1, "D")).astype(object).month)
        elif group == "date_bounds":
            month = int(value[0][:2])
        else:
            raise ValueError(f"Unknown group `{group}`.")
        freq = "YS-" + _MONTH_ABBREVIATIONS[month]
    return freq


def cumulative_difference(data, threshold, op, freq=None):
    """Sum of the excess over (deficit under) a threshold -- indices/generic.py:1514-1552."""
    code = get_op(op, constrain=(">", ">=", "<", "<="))
    thr = threshold_in_units_of(threshold, data) if isinstance(threshold, str) else float(threshold)
    x2d, cell_shape, other, ta = _unwrap(data)      # freq=None: the whole series (one period, no time dim)
    out, _ = device.period_reduce(x2d, ta.period_offsets(freq), _lib.STATS["sum"], _lib.TF_EXCESS, code, thr)
    attrs = attrs_of(data)
    u = attrs.get("units", "")
    attrs["units"] = f"{u} d".strip()
    return _wrap_periods(data, out, cell_shape, other, ta, freq, attrs)


# --------------------------------------------------------------------------------- a5/a6 spells
def spell_length_statistics(data, threshold, window, win_reducer, op, spell_reducer, freq, min_gap=1,
                            resample_before_rl=True, **indexer):
    """Statistics of spell lengths -- indices/generic.py:588-686 (-> 543-585).

    ``window == 1`` (the maximum_consecutive_dry/wet_days family) is one fused kernel:
    compare -> run-length state machine -> reducer, per (period, cell).
    """
    if indexer and (min_gap > 1):
        raise NotImplementedError("select_time indexers together with min_gap > 1 are not supported")
    if min_gap < 1:
        raise ValueError("min_gap must be >= 1")
    if min_gap > 1 and not resample_before_rl:
        raise NotImplementedError("min_gap > 1 is supported with resample_before_rl=True only")
    code = get_op(op)
    thr = threshold_in_units_of(threshold, data) if isinstance(threshold, str) else _scalar_threshold(threshold)[0]
    reducers = [spell_reducer] if isinstance(spell_reducer, str) else list(spell_reducer)
    x2d, cell_shape, other, ta = _unwrap(data)
    poff = ta.period_offsets(freq)
    sel_mask = None
    if indexer:
        # is_in_spell = select_time(spell_mask(...), **indexer)  (indices/generic.py:557-558): the mask is built
        # on the whole series, masked (NaN) out of season, and the run statistics run on it with `mask > 0`
        keep = ta.select_mask(**indexer).astype(np.uint8)
        starts = np.zeros(len(ta), bool)
        starts[np.asarray(poff[:-1])] = True
        first_in = keep.astype(bool) & ~np.concatenate([[True], keep[:-1].astype(bool)])
        keep[first_in & ~(starts if resample_before_rl else np.zeros(len(ta), bool))] = 2
        if not resample_before_rl:
            keep[0] = min(keep[0], 1)
        wstat = _lib.STATS[(win_reducer or "sum").replace("integral", "sum")]
        sel_mask = device.spell_mask(x2d, window, wstat, code, thr, keep,
                                     drop_nan_adjacent=(OPTIONS["rle_nan_adjacent"] == "drop"))
    gap_mask = None
    if min_gap > 1 and window > 1:
        # spell_mask(window > 1) materialised once (indices/generic.py:519-535), then runs_with_holes + the run
        # statistics on it (:537-538, 557-585): the window-1 min_gap kernel on the 0/1 mask
        if win_reducer not in ("min", "max", "sum", "mean"):
            raise ValueError(f"win_reducer must be one of min, max, sum, mean; got {win_reducer!r}")
        gap_mask = device.spell_mask(x2d, window, _lib.STATS[win_reducer], code, thr)
    outs = []
    for sr in reducers:
        if sr not in _lib.RL_REDUCERS:
            raise NotImplementedError(f"spell reducer {sr!r} is not supported by the xclim_b200 hot path")
        if gap_mask is not None:
            out = device.period_runstat_gap(gap_mask, poff, _lib.OPS[">"], 0.5, _lib.RL_REDUCERS[sr], min_gap)
        elif sel_mask is not None:
            out, _ = device.period_runstat(sel_mask, poff, _lib.OPS[">"], 0.0, _lib.RL_REDUCERS[sr], 1, resample_before_rl)
        elif window == 1 and min_gap > 1:     # runs_with_holes (indices/generic.py:537-538)
            out = device.period_runstat_gap(x2d, poff, code, thr, _lib.RL_REDUCERS[sr], min_gap)
        elif window == 1:
            out, _ = device.period_runstat(x2d, poff, code, thr, _lib.RL_REDUCERS[sr], 1, resample_before_rl)
        else:
            # rolling-window spell masks (indices/generic.py:434-585 for window > 1)
            if win_reducer not in ("min", "max", "sum", "mean"):
                raise ValueError(f"win_reducer must be one of min, max, sum, mean; got {win_reducer!r}")
            out = device.spell_runstat(x2d, poff, window, _lib.STATS[win_reducer], code, thr, _lib.RL_REDUCERS[sr],
                                       resample_before_rl)
        attrs = attrs_of(data)
        attrs["units"] = "" if sr == "count" else "d"
        outs.append(_wrap_periods(data, out, cell_shape, other, ta, freq, attrs, dtype=np.float32))
    return outs[0] if len(outs) == 1 else tuple(outs)


# --------------------------------------------------------------------------------- a4 rolling + resample
def select_rolling_resample_op(da, op, window, window_center=True, window_op="mean", freq="YS", out_units=None,
                               **indexer):
    """Rolling window statistic, then per-period reduction -- indices/generic.py:128-174."""
    wop = window_op.replace("integral", "sum")
    if wop not in ("sum", "mean", "min", "max"):
        raise NotImplementedError(f"rolling window_op {window_op!r} is not supported by the xclim_b200 hot path")
    if not isinstance(op, str) or op not in _lib.STATS:
        raise NotImplementedError(f"resample op {op!r} is not supported by the xclim_b200 hot path")
    x2d, cell_shape, other, ta = _unwrap(da)
    if indexer:
        # the reference selects AFTER rolling (indices/generic.py:169-174): rolling on the full series, then
        # select_time on the rolled values -- a mask on the window LABELS
        out = device.rolling_period_reduce_sel(x2d, ta.period_offsets(freq), window, _lib.STATS[wop], window_center,
                                               _lib.STATS[op], ta.select_mask(**indexer))
    else:
        out = device.rolling_period_reduce(x2d, ta.period_offsets(freq), window, _lib.STATS[wop], window_center,
                                           _lib.STATS[op])
    attrs = attrs_of(da)
    if out_units is not None:
        attrs["units"] = out_units
    return _wrap_periods(da, out, cell_shape, other, ta, freq, attrs)


def statistics(data, reducer, freq):
    """indices/generic.py:1255-1275."""
    out = select_resample_op(data, reducer, freq)
    return out.assign_attrs(units=attrs_of(data).get("units", ""))


def thresholded_statistics(data, op, threshold, reducer, freq, constrain=None):
    """Statistic of the values fulfilling ``data op threshold`` -- indices/generic.py:1278-1320."""
    code = get_op(op, constrain)
    thr = threshold_in_units_of(threshold, data) if isinstance(threshold, str) else float(threshold)
    if reducer not in ("max", "min", "mean", "sum"):
        raise NotImplementedError(f"reducer {reducer!r} is not supported")
    x2d, cell_shape, other, ta = _unwrap(data)
    out, _ = device.period_reduce(x2d, ta.period_offsets(freq), _lib.STATS[reducer], _lib.TF_WHERE, code, thr)
    return _wrap_periods(data, out, cell_shape, other, ta, freq, attrs_of(data))


def temperature_sum(data, op, threshold, freq):
    """indices/generic.py:1323-1357: sum of (data - threshold) where the condition holds, sign-flipped
    for < / <= -- numerically the clipped difference of :func:`cumulative_difference`."""
    return cumulative_difference(data, threshold, op, freq)


def count_occurrences(data, threshold, freq, op, constrain=None):
    """indices/generic.py:960-999."""
    thr = threshold_in_units_of(threshold, data) if isinstance(threshold, str) else threshold
    out = threshold_count(data, op, thr, freq, constrain)
    return out.assign_attrs(units="d")


def _occurrence(data, threshold, freq, op, constrain, last):
    from .run_length import index_to_doy
    import torch
    code = get_op(op, constrain)
    thr, f64 = (threshold_in_units_of(threshold, data), False) if isinstance(threshold, str) else \
        _scalar_threshold(threshold)
    x2d, cell_shape, other, ta = _unwrap(data)
    poff = ta.period_offsets(freq)
    idx = device.period_boundary_run(x2d, poff, code, thr, 1, last=last, cmp_f64=f64)
    out = index_to_doy(idx.to(torch.float64), poff, ta)      # coord="dayofyear" (core/utils.py:202-276)
    attrs = attrs_of(data)
    attrs.update(units="", is_dayofyear=np.int32(1), calendar=ta.calendar)
    return _wrap_periods(data, out, cell_shape, other, ta, freq, attrs, dtype=np.float64)


def first_occurrence(data, threshold, freq, op, constrain=None):
    """Day of year of the first step of each period where ``data op threshold`` -- indices/generic.py:
    1107-1156 (``rl.first_run(cond, window=1, coord="dayofyear")`` per group; NaN when there is none --
    or, by the argmax == argmin rule of the reference, when every step qualifies)."""
    return _occurrence(data, threshold, freq, op, constrain, last=False)


def last_occurrence(data, threshold, freq, op, constrain=None):
    """indices/generic.py:1159-1206."""
    return _occurrence(data, threshold, freq, op, constrain, last=True)


def count_level_crossings(low_data, high_data, threshold, freq, *, op_low="<", op_high=">="):
    """Days on which ``low_data`` is under and ``high_data`` over the same threshold --
    indices/generic.py:917-957 (both variables in the same units)."""
    from .units import units_of
    if units_of(high_data) != units_of(low_data):
        raise NotImplementedError("count_level_crossings: give both variables in the same units")
    return bivariate_count_occurrences(data_var1=low_data, data_var2=high_data, threshold_var1=threshold,
                                       threshold_var2=threshold, freq=freq, op_var1=op_low, op_var2=op_high,
                                       var_reducer="all", constrain_var1=("<", "<="), constrain_var2=(">", ">="))


# --------------------------------------------------------------------------------- detrend
def detrend(ds, dim="time", deg=1):
    """``ds`` minus its polynomial trend of degree ``deg`` along time -- indices/generic.py:1711-1736 (``polyfit``
    then ``polyval``, ``ds - trend`` with the attributes kept).  The trend of each cell is the least-squares
    polynomial over its valid steps (a gap-free daily axis); the result is float64, as float32 data minus the
    float64 trend is in the reference, and NaN where ``ds`` is NaN.  DataArray / Field inputs, ``dim="time"`` and
    degrees 0 to 2 only."""
    from .field import Field
    if not (isinstance(ds, Field) or is_xarray(ds)):
        raise NotImplementedError(f"detrend takes a DataArray or a Field, got {type(ds).__name__}")
    if dim != "time":
        raise NotImplementedError("detrend along a dimension other than time is not supported")
    if isinstance(deg, bool) or not isinstance(deg, (int, np.integer)) or deg < 0:
        raise ValueError(f"deg must be a non-negative integer, got {deg!r}")
    if deg > 2:
        raise NotImplementedError(f"deg={deg}: only polynomial degrees 0, 1 and 2 are supported")
    dims = dims_of(ds)
    x2d, cell_shape, other, ta = _unwrap(ds)
    out = device.detrend(x2d, int(deg))
    vals = np.moveaxis(out.reshape((out.shape[0],) + cell_shape).cpu().numpy(), 0, dims.index("time"))
    return wrap_like(ds, vals, dims, time=ta if ta.coord is None else ta.coord, attrs=attrs_of(ds),
                     name=getattr(ds, "name", None))


# --------------------------------------------------------------------------------- a12 seasons / dates
def season(data, thresh, window, op, stat, freq, mid_date=None, constrain=None):
    """Season start / end (day of year) or length -- indices/generic.py:769-853 (+ run_length.py:891-1145)."""
    from . import seasons
    code = get_op(op, constrain)
    if stat not in ("start", "end", "length"):
        raise ValueError(f"stat must be 'start', 'end' or 'length', got {stat!r}")
    thr = threshold_in_units_of(thresh, data) if isinstance(thresh, str) else float(thresh)
    x2d, cell_shape, other, ta = _unwrap(data)
    out = seasons.season(x2d, ta, freq, code, thr, window, mid_date, stat)
    attrs = attrs_of(data)
    if stat == "length":
        attrs["units"] = "d"
    else:
        attrs.update(units="", is_dayofyear=np.int32(1), calendar=ta.calendar)
    return _wrap_periods(data, out, cell_shape, other, ta, freq, attrs, dtype=np.float64)


def first_day_threshold_reached(data, *, threshold, op, after_date, window=1, freq="YS", constrain=None):
    """indices/generic.py:1555-1608: day of year of the first run of `window` steps after a date."""
    from . import seasons
    code = get_op(op, constrain)
    thr = threshold_in_units_of(threshold, data) if isinstance(threshold, str) else float(threshold)
    x2d, cell_shape, other, ta = _unwrap(data)
    out = seasons.first_run_after_date(x2d, ta, freq, code, thr, window, after_date)
    attrs = attrs_of(data)
    attrs.update(units="", is_dayofyear=np.int32(1), calendar=ta.calendar)
    return _wrap_periods(data, out, cell_shape, other, ta, freq, attrs, dtype=np.float64)


def bivariate_count_occurrences(*, data_var1, data_var2, threshold_var1, threshold_var2, freq, op_var1, op_var2,
                                var_reducer, constrain_var1=None, constrain_var2=None):
    """indices/generic.py:1002-1073: count of steps where both ("all") or either ("any") condition holds."""
    if var_reducer not in ("all", "any"):
        raise ValueError(f"Unsupported value for var_reducer: {var_reducer}")
    c1, c2 = get_op(op_var1, constrain_var1), get_op(op_var2, constrain_var2)
    t1 = threshold_in_units_of(threshold_var1, data_var1) if isinstance(threshold_var1, str) else float(threshold_var1)
    t2 = threshold_in_units_of(threshold_var2, data_var2) if isinstance(threshold_var2, str) else float(threshold_var2)
    x1, cell_shape, other, ta = _unwrap(data_var1)
    x2, cs2, _, _ = _unwrap(data_var2)
    if cs2 != cell_shape:
        raise ValueError("the two variables must share the same grid")
    out = device.period_runstat2(x1, x2, ta.period_offsets(freq), c1, t1, c2, t2, _lib.RL_REDUCERS["sum"], 1, True,
                                 var_any=(var_reducer == "any"))
    attrs = attrs_of(data_var1)
    attrs["units"] = "d"
    return _wrap_periods(data_var1, out, cell_shape, other, ta, freq, attrs, dtype=np.int64)
