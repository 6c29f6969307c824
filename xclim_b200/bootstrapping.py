"""CUDA implementation behind ``xclim.core.bootstrapping`` (percentile bootstrap, Zhang 2005)."""
from __future__ import annotations

import numpy as np

from . import _lib, device
from .calendar import adjust_table, table_on_device
from .field import attrs_of
from .generic import _unwrap, _wrap_periods


def bootstrap_doy_count(da, per, freq, op, constrain):
    """Body of ``percentile_bootstrap`` for the doy-percentile day counts (tx90p & family) --
    core/bootstrapping.py:81-211.  Error behaviour follows the reference: ``KeyError`` when the
    percentile array was not made by ``percentile_doy`` (:131-143) or when the base period covers
    all / none of the studied period (:159-168)."""
    code = _lib.op_code(op, constrain)
    pattrs = attrs_of(per)
    if "percentile_doy" not in pattrs.get("history", ""):
        raise KeyError("`bootstrap` can only be used with percentiles computed using `percentile_doy`")
    clim = pattrs["climatology_bounds"]
    window, alpha, beta = int(pattrs["window"]), float(pattrs["alpha"]), float(pattrs["beta"])
    pcs = np.atleast_1d(np.asarray(per.coords["percentiles"] if "percentiles" in getattr(per, "coords", {}) else
                                   pattrs.get("percentiles")))
    if pcs.size != 1:
        raise ValueError("select one percentile first: per.sel(percentiles=p)")
    percentile = float(pcs[0])
    x2d, cell_shape, other, ta = _unwrap(da)
    sl = ta.sel_dates(str(clim[0])[:10], str(clim[1])[:10])    # da.sel(time=slice(*clim))  (:158): full dates
    n_over = sl.stop - sl.start
    if n_over == len(ta):
        raise KeyError("`bootstrap` is unnecessary when all years are overlapping between reference "
                       "(percentiles period) and studied (index period) periods")
    if n_over == 0:
        raise KeyError("`bootstrap` is unnecessary when no year overlap between reference "
                       "(percentiles period) and studied (index period) periods.")
    gid = ta.bootstrap_group_ids(freq)                        # year groups (:175, 214-223)
    base_gid = gid[sl]
    groups, starts, lens = np.unique(base_gid, return_index=True, return_counts=True)
    L, N = int(lens[0]), len(groups)
    if N < 2:
        raise KeyError("`bootstrap` needs at least two years in the reference period")
    poff = ta.period_offsets(freq)
    P = len(poff) - 1
    pidx = np.repeat(np.arange(P), np.diff(poff))             # period of every step
    step_period = pidx[sl].astype(np.int32)
    if len(set(lens.tolist())) == 1:
        boot = device.bootstrap_doy_count(x2d, sl.start, N, L, step_period, P, window, percentile, alpha, beta, code)
    else:
        boot = _bootstrap_unequal_blocks(x2d, ta, sl, starts, lens, poff, step_period, window, percentile, alpha,
                                         beta, code)
    # periods outside the base: plain count against the original table (:205-207)
    from .indices import _table_in_units_of          # convert_units_to(per, da): indices/_multivariate.py:1583
    table = _table_in_units_of(table_on_device(per, cell_shape, other, x2d.device), per, da)
    table, doy_idx = adjust_table(table, ta)
    plain, _ = device.doy_threshold_count(x2d, poff, doy_idx, table, code)
    in_base = np.zeros(P, bool)
    in_base[np.unique(step_period)] = True
    import torch
    mask = torch.from_numpy(in_base).to(x2d.device)[:, None]
    out = torch.where(mask, boot, plain.to(torch.float64))
    attrs = attrs_of(da)
    attrs["units"] = "d"
    return _wrap_periods(da, out, cell_shape, other, ta, freq, attrs, dtype=np.float64)


def replacement_rows(ta_base, starts, lens, yi, si):
    """Rows (relative to the base slice) whose values stand in for block ``yi`` when it is replaced
    by block ``si`` -- core/bootstrapping.py:255-279.  ``-1`` = missing (NaN).  ``None`` = the
    reference leaves the block untouched (:257-260)."""
    ly, ls = int(lens[yi]), int(lens[si])
    src = int(starts[si]) + np.arange(ls)
    if ls < 360 and ls < ly:                                   # partial first / last anchored year
        return None
    if ls == ly:
        return src
    feb29 = lambda a, n: np.nonzero((ta_base.month[a:a + n] == 2) & (ta_base.day[a:a + n] == 29))[0]
    if ly == 365:                                              # source.convert_calendar("noleap"): drop Feb 29
        hit = feb29(int(starts[si]), ls)
        if ls == 366 and hit.size == 1:
            return np.delete(src, hit[0])
    elif ly == 366:                                            # convert_calendar("366_day", missing=NaN)
        hit = feb29(int(starts[yi]), ly)
        if ls == 365 and hit.size == 1:
            return np.insert(src, hit[0], -1)
    elif ly < 365 and ls >= ly:                                # source.data[:len(bloc)]
        return src[:ly]
    raise NotImplementedError(f"bootstrap: cannot map a block of {ls} steps onto a block of {ly} steps")


def _bootstrap_unequal_blocks(x2d, ta, sl, starts, lens, poff, step_period, window, percentile, alpha, beta, code):
    """Year blocks of unequal length (standard / proleptic_gregorian calendars): every replacement
    (in-base year y <- base year s, 365 <-> 366 conversion of core/bootstrapping.py:266-269) is a
    virtual-row map of the base series, so the percentile kernels run on the ORIGINAL rows
    (``xc_percentile_doy_vrow_f32``); the counts of year y against each of the N-1 tables are summed
    as integers and divided once.  N(N-1) table builds: slower than the fused equal-length kernel
    (which shares the per-day sorted extremes between all replacements) but exact and copy-free."""
    import torch
    from .calendar import year_ordinals
    ta_b = ta.isel(sl)
    xb = x2d[sl.start:sl.stop]
    yidx, years = year_ordinals(ta_b)
    n_doy = int(ta_b.doy.max())
    Tb, C = xb.shape
    P = len(poff) - 1
    N = len(starts)
    acc = torch.zeros((P, C), dtype=torch.int64, device=x2d.device)
    nrep = np.zeros(P, dtype=np.int64)
    ident = np.arange(Tb, dtype=np.int32)
    for yi in range(N):
        a, n = int(starts[yi]), int(lens[yi])
        periods = np.unique(step_period[a:a + n])              # periods of the studied axis inside block y
        p0, p1 = int(periods[0]), int(periods[-1]) + 1
        sub_off = (poff[p0:p1 + 1] - poff[p0]).astype(np.int32)
        xs = x2d[poff[p0]:poff[p1]]
        ta_s = ta.isel(slice(int(poff[p0]), int(poff[p1])))
        for si in range(N):
            if si == yi:
                continue
            rows = replacement_rows(ta_b, starts, lens, yi, si)
            vrow = ident
            if rows is not None:
                vrow = ident.copy()
                vrow[a:a + n] = rows
            table = device.percentile_doy(xb, ta_b.doy, yidx, n_doy, len(years), window, [percentile], alpha, beta,
                                          vrow=vrow)[0]
            if n_doy == 366:                                   # core/calendar.py:484-485
                table = device.doy_interp(table[:365].contiguous(), 1, 366)
            table, doy_idx = adjust_table(table, ta_s)
            cnt, _ = device.doy_threshold_count(xs, sub_off, doy_idx, table, code)
            acc[p0:p1] += cnt.to(torch.int64)
            nrep[p0:p1] += 1
    div = torch.from_numpy(np.maximum(nrep, 1)).to(x2d.device).to(torch.float64)[:, None]
    return acc.to(torch.float64) / div
