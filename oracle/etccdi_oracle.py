"""CPU oracle for the remaining ETCCDI day-of-year percentile indices, the compound percentile days and the daily
temperature range.  TEST INFRASTRUCTURE ONLY (see xclim_oracle.py for the conventions: arrays are ``(time, ...)``,
``poff`` the P + 1 period boundaries, ``doy`` the ``time.dt.dayofyear`` values, tables ``(n_doy, ...)``).

Every function restates reference code in numpy, citing ``file:line`` relative to ``/root/reference/src/xclim``.
"""
from __future__ import annotations

import numpy as np

from oracle import xclim_oracle as O


def _spell_duration(x, table, doy, poff, window, resample_before_rl, op, constrain, cal_max_doy):
    thresh = O.resample_doy(table, doy, cal_max_doy)
    cond = O.compare(x, op, thresh, constrain)                     # float32 data against float64 thresholds
    out = O.resample_and_rl(cond, resample_before_rl, O.windowed_run_count, window, poff=poff)
    return np.asarray(out, dtype=np.float32)                       # to_agg_units(..., "count") of daily data


def warm_spell_duration_index(tasmax, table, doy, poff, window=6, resample_before_rl=True, op=">", cal_max_doy=None):
    """indices/_multivariate.py:1780-1795."""
    return _spell_duration(tasmax, table, doy, poff, window, resample_before_rl, op, (">", ">="), cal_max_doy)


def cold_spell_duration_index(tasmin, table, doy, poff, window=6, resample_before_rl=True, op="<", cal_max_doy=None):
    """indices/_multivariate.py:138-153."""
    return _spell_duration(tasmin, table, doy, poff, window, resample_before_rl, op, ("<", "<="), cal_max_doy)


def fraction_over_precip_thresh(pr, pr_per, thresh, poff, op=">", doy=None, cal_max_doy=None):
    """indices/_multivariate.py:1283-1297.  ``pr_per``: (n_doy, ...) with ``doy`` (a day-of-year table), else one
    value per cell ``(...)``; ``thresh`` a Python float in pr's units.  The sums are float32, as xarray's
    ``resample().sum()`` of float32 data returns them."""
    pr = np.asarray(pr, dtype=np.float32)
    pr_per = np.asarray(pr_per, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        tp = np.where(pr_per > thresh, pr_per, thresh)             # pr_per.where(pr_per > thresh, thresh)
    if doy is not None:
        tp = O.resample_doy(tp, doy, cal_max_doy)
    constrain = (">", ">=")
    total = np.where(O.compare(pr, op, thresh, constrain), pr, np.float32(0))
    over = np.where(O.compare(pr, op, tp, constrain), pr, np.float32(0))
    total = np.stack([total[s:e].sum(axis=0, dtype=np.float64) for s, e in O._groups(poff)]).astype(np.float32)
    over = np.stack([over[s:e].sum(axis=0, dtype=np.float64) for s, e in O._groups(poff)]).astype(np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        return over / total


_COMPOUND = {"cold_and_dry_days": ("<", "<"), "warm_and_dry_days": (">", "<"), "warm_and_wet_days": (">", ">"),
             "cold_and_wet_days": ("<", ">")}


def compound_days(name, tas, pr, tas_table, pr_table, doy, poff, cal_max_doy=None):
    """indices/_multivariate.py:162-416: ``np.logical_and(tas op1 tas_per[doy], pr op2 pr_per[doy])`` summed per
    period (both compares in float64)."""
    op1, op2 = _COMPOUND[name]
    c1 = O.compare(tas, op1, O.resample_doy(tas_table, doy, cal_max_doy))
    c2 = O.compare(pr, op2, O.resample_doy(pr_table, doy, cal_max_doy))
    both = np.logical_and(c1, c2)
    return np.stack([both[s:e].sum(axis=0) for s, e in O._groups(poff)]).astype(np.int64)


def daily_temperature_range(tasmin, tasmax, poff, op="mean"):
    """indices/_multivariate.py:552-557: ``select_resample_op(tasmax - tasmin, op)``, the difference in float32."""
    dtr = np.asarray(tasmax, dtype=np.float32) - np.asarray(tasmin, dtype=np.float32)
    return O.resample_reduce(dtr, poff, op).astype(np.float32)


def daily_temperature_range_variability(tasmin, tasmax, poff):
    """indices/_multivariate.py:593-598: ``abs((tasmax - tasmin).diff("time"))`` labelled with the later step
    (xarray's ``diff(label="upper")``), then the per-period mean.  The first step has no difference: a period
    holding only it is NaN."""
    dtr = np.asarray(tasmax, dtype=np.float32) - np.asarray(tasmin, dtype=np.float32)
    vdtr = np.full_like(dtr, np.nan)
    vdtr[1:] = np.abs(dtr[1:] - dtr[:-1])
    return O.resample_reduce(vdtr, poff, "mean").astype(np.float32)
