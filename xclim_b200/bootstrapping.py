"""CUDA implementation behind ``xclim.core.bootstrapping`` (percentile bootstrap, Zhang 2005)."""
from __future__ import annotations

import numpy as np

from . import _lib, device
from .calendar import adjust_table, table_on_device
from .field import attrs_of
from .generic import _unwrap, _wrap_periods


class BootstrapPercentileError(KeyError, NotImplementedError):
    """``bootstrap=True`` with a percentile table that ``percentile_doy`` did not make (core/bootstrapping.py:
    131-143 raises ``KeyError``).  Also a ``NotImplementedError``: the indices that had no bootstrap raised that
    for every ``bootstrap=True`` call."""


def _check_provenance(per):
    """core/bootstrapping.py:131-143, the first check of ``percentile_bootstrap``, before any device call."""
    if "percentile_doy" not in attrs_of(per).get("history", ""):
        raise BootstrapPercentileError("`bootstrap` can only be used with percentiles computed using `percentile_doy`")


class _Setup:
    """The bookkeeping every bootstrapped index shares (core/bootstrapping.py:128-180): the table's percentile
    parameters, the base slice, the bootstrap year groups and the output period of every base step."""

    def __init__(self, da, per, freq):
        _check_provenance(per)
        pattrs = attrs_of(per)
        self.clim = pattrs["climatology_bounds"]
        self.window, self.alpha, self.beta = int(pattrs["window"]), float(pattrs["alpha"]), float(pattrs["beta"])
        pcs = np.atleast_1d(np.asarray(per.coords["percentiles"] if "percentiles" in getattr(per, "coords", {}) else
                                       pattrs.get("percentiles")))
        if pcs.size != 1:
            raise ValueError("select one percentile first: per.sel(percentiles=p)")
        self.percentile = float(pcs[0])
        self.x2d, self.cell_shape, self.other, self.ta = _unwrap(da)
        ta = self.ta
        sl = ta.sel_dates(str(self.clim[0])[:10], str(self.clim[1])[:10])   # da.sel(time=slice(*clim)) (:158)
        n_over = sl.stop - sl.start
        if n_over == len(ta):
            raise KeyError("`bootstrap` is unnecessary when all years are overlapping between reference "
                           "(percentiles period) and studied (index period) periods")
        if n_over == 0:
            raise KeyError("`bootstrap` is unnecessary when no year overlap between reference "
                           "(percentiles period) and studied (index period) periods.")
        self.sl = sl
        self.gid = ta.bootstrap_group_ids(freq)                      # year groups (:175, 214-223)
        groups, starts, lens = np.unique(self.gid[sl], return_index=True, return_counts=True)
        self.starts, self.lens = starts, lens
        self.L, self.N = int(lens[0]), len(groups)
        if self.N < 2:
            raise KeyError("`bootstrap` needs at least two years in the reference period")
        self.poff = ta.period_offsets(freq)
        self.P = len(self.poff) - 1
        pidx = np.repeat(np.arange(self.P), np.diff(self.poff))      # period of every step
        self.step_period = pidx[sl].astype(np.int32)
        self.equal = len(set(lens.tolist())) == 1
        self.in_base = np.zeros(self.P, bool)
        self.in_base[np.unique(self.step_period)] = True
        self.freq = freq

    def labelled_blocks(self):
        """The base blocks that are bootstrapped as the reference decides it (core/bootstrapping.py:182-184): a
        year group of the series is bootstrapped when its LABEL year is a year of the base, and then over the
        whole group, steps outside the base included.  Returns ``[(block, p0, p1)]`` with the group's periods
        [p0, p1), and sets ``in_base`` to those periods.  With an anchored ``freq`` this differs from "the periods
        that hold base steps": YS-JUL's group labelled with the year before the base is not bootstrapped, and
        QS-DEC's group of the last base December is, into the next year."""
        ta = self.ta
        bfreq = ta.bootstrap_freq(self.freq)
        gpoff = ta.period_offsets(bfreq)
        glabel = np.array([int(lab[:4]) for lab in ta.period_labels(bfreq)])
        gidx = np.repeat(np.arange(len(gpoff) - 1), np.diff(gpoff))     # group of every step, in time order
        base_years = set(np.asarray(ta.year[self.sl.start:self.sl.stop]).tolist())
        blocks = []
        self.in_base = np.zeros(self.P, bool)
        for yi, a in enumerate(self.starts):
            g = int(gidx[self.sl.start + int(a)])
            if int(glabel[g]) not in base_years:
                continue
            p0, p1 = np.searchsorted(self.poff, [gpoff[g], gpoff[g + 1]])
            blocks.append((yi, int(p0), int(p1)))
            self.in_base[p0:p1] = True
        # the fused kernels: every block a whole group of the series, of one length, and bootstrapped
        whole = all(int(gpoff[g + 1] - gpoff[g]) == int(n) for g, n in
                    zip(gidx[self.sl.start + self.starts], self.lens))
        self.equal = self.equal and whole and len(blocks) == self.N
        return blocks

    def merge(self, da, boot, plain, freq, units, dtype):
        """Bootstrapped values for the in-base periods, ``plain`` for the others (:205-207), wrapped like da."""
        import torch
        mask = torch.from_numpy(self.in_base).to(self.x2d.device)[:, None]
        out = torch.where(mask, boot, plain.to(boot.dtype))
        attrs = attrs_of(da)
        attrs["units"] = units
        return _wrap_periods(da, out, self.cell_shape, self.other, self.ta, freq, attrs, dtype=dtype)

    def table(self, per, da, floor=None):
        """The original table in da's units (convert_units_to(per, da), indices/_multivariate.py:1583), floored
        like the index does, and the table row of every step."""
        import torch
        from .indices import _table_in_units_of
        table = _table_in_units_of(table_on_device(per, self.cell_shape, self.other, self.x2d.device), per, da)
        if floor is not None:
            table = torch.where(table > floor, table, torch.full_like(table, floor))
        return adjust_table(table, self.ta)


def bootstrap_doy_count(da, per, freq, op, constrain):
    """Body of ``percentile_bootstrap`` for the doy-percentile day counts (tx90p & family) --
    core/bootstrapping.py:81-211.  Error behaviour follows the reference: ``KeyError`` when the
    percentile array was not made by ``percentile_doy`` (:131-143) or when the base period covers
    all / none of the studied period (:159-168)."""
    code = _lib.op_code(op, constrain)
    b = _Setup(da, per, freq)
    if b.equal:
        boot = device.bootstrap_doy_count(b.x2d, b.sl.start, b.N, b.L, b.step_period, b.P, b.window, b.percentile,
                                          b.alpha, b.beta, code)
    else:
        boot = _bootstrap_unequal_blocks(
            b.x2d, b.ta, b.sl, b.starts, b.lens, b.poff, b.step_period, b.window, b.percentile, b.alpha, b.beta,
            lambda xs, off, doy_idx, table: device.doy_threshold_count(xs, off, doy_idx, table, code)[0])
    # periods outside the base: plain count against the original table (:205-207)
    table, doy_idx = b.table(per, da)
    plain, _ = device.doy_threshold_count(b.x2d, b.poff, doy_idx, table, code)
    return b.merge(da, boot, plain, freq, "d", np.float64)


def _nested(b, freq):
    """The output periods must nest in the bootstrap year groups (weekly / daily periods do not)."""
    first = b.gid[b.poff[:-1]]
    last = b.gid[b.poff[1:] - 1]
    if not np.array_equal(first, last):
        raise NotImplementedError(f"bootstrap with freq={freq!r}: its periods do not nest in the bootstrap years")


def bootstrap_doy_index(da, per, freq, op, constrain, kind, window=1, resample_before_rl=True, floor=None):
    """``percentile_bootstrap`` (core/bootstrapping.py:81-211) on the indices whose value depends on the order of
    the days over the threshold or on their values: ``kind`` "spell" (warm / cold spell duration index,
    indices/_multivariate.py:69-153, 1719-1795, ``window`` and ``resample_before_rl``), "count"
    (days_over_precip_thresh, :1174-1233) or "sum" (fraction_over_precip_thresh, :1238-1297), the last two with
    the wet-day threshold ``floor`` in da's units.

    As in the reference, every bootstrap year is computed on its own slice of the series, so runs end at the edges
    of the bootstrap years, outside the base too; and the altered tables are percentiles of ``da`` itself (dry days
    included for precipitation) whatever series ``per`` was computed from."""
    import torch
    _check_provenance(per)
    code = _lib.op_code(op, constrain)
    b = _Setup(da, per, freq)
    _nested(b, freq)
    blocks = b.labelled_blocks()
    table, doy_idx = b.table(per, da, floor)
    # the original table: out-of-base periods (:205-207), and the wet-day totals of the fraction
    wet = None
    if kind == "spell":
        plain = _spells_per_year(b, doy_idx, table, code, window, resample_before_rl)
    elif kind == "count":
        plain = device.doy_threshold_count(b.x2d, b.poff, doy_idx, table, code)[0]
    else:
        s_thr, wet = device.period_sums_thr(b.x2d, b.poff, code, table, floor, doy_index=doy_idx)
        plain = s_thr / wet
    if b.equal:
        boot, _ = device.bootstrap_doy_index(b.x2d, b.sl.start, b.N, b.L, b.step_period, b.P, b.window,
                                             b.percentile, b.alpha, b.beta, code, kind, window, resample_before_rl,
                                             floor, wet)
    else:
        boot = _bootstrap_unequal_blocks(b.x2d, b.ta, b.sl, b.starts, b.lens, b.poff, b.step_period, b.window,
                                         b.percentile, b.alpha, b.beta,
                                         _replacement_index(kind, code, window, resample_before_rl, floor, wet),
                                         fraction=kind == "sum", blocks=blocks)
    if kind == "sum":
        return b.merge(da, boot, plain, freq, "", np.float32)
    return b.merge(da, boot, plain.to(torch.float64), freq, "d", np.float64)


def _spells_per_year(b, doy_idx, table, code, window, resample_before_rl):
    """The spell index against the original table, each bootstrap year on its own slice (core/bootstrapping.py:
    182-207 applies the index to ``da.isel(time=year_slice)``): runs end at the year edges.  With
    resample_before_rl the periods already end there, and one call does."""
    import torch
    red = _lib.RL_REDUCERS["sum"]
    if resample_before_rl:
        return device.doy_runstat(b.x2d, b.poff, doy_idx, table, code, red, window, True)[0]
    doy_idx = np.asarray(doy_idx)
    out = []
    _, gstart = np.unique(b.gid, return_index=True)
    edges = np.append(np.sort(gstart), len(b.ta))
    for a, e in zip(edges[:-1], edges[1:]):
        p0, p1 = np.searchsorted(b.poff, a), np.searchsorted(b.poff, e)
        off = (b.poff[p0:p1 + 1] - a).astype(np.int32)
        out.append(device.doy_runstat(b.x2d[a:e], off, doy_idx[a:e], table, code, red, window, False)[0])
    return torch.cat(out, 0)


def _replacement_index(kind, code, window, resample_before_rl, floor, wet):
    """The index of one bootstrap year's slice against one altered table, for _bootstrap_unequal_blocks."""
    import torch
    if kind == "spell":
        red = _lib.RL_REDUCERS["sum"]
        return lambda xs, off, doy_idx, table: device.doy_runstat(xs, off, doy_idx, table, code, red, window,
                                                                  resample_before_rl)[0].to(torch.int64)
    tp = lambda table: torch.where(table > floor, table, torch.full_like(table, floor))  # noqa: E731
    if kind == "count":
        return lambda xs, off, doy_idx, table: device.doy_threshold_count(xs, off, doy_idx, tp(table), code)[0]

    def fraction(xs, off, doy_idx, table, p0):
        s_thr, _ = device.period_sums_thr(xs, off, code, tp(table), floor, doy_index=doy_idx)
        return s_thr / wet[p0:p0 + len(off) - 1]
    fraction.takes_p0 = True
    return fraction


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


def _bootstrap_unequal_blocks(x2d, ta, sl, starts, lens, poff, step_period, window, percentile, alpha, beta, index,
                              fraction=False, blocks=None):
    """Year blocks of unequal length (standard / proleptic_gregorian calendars): every replacement
    (in-base year y <- base year s, 365 <-> 366 conversion of core/bootstrapping.py:266-269) is a
    virtual-row map of the base series, so the percentile kernels run on the ORIGINAL rows
    (``xc_percentile_doy_vrow_f32``); ``index(xs, offsets, doy_idx, table)`` then computes the index of year y's
    slice against each of the N-1 tables.  Integer results are summed and divided once; with ``fraction`` the
    float32 results are averaged by the rule of xc_bootstrap_doy_index_f32 (float64 sum of the non-NaN terms in s
    order over their number, rounded once).  ``blocks``: the (block, p0, p1) to bootstrap over the periods
    [p0, p1) (default: every block over the periods holding its steps).  N(N-1) table builds: slower than the fused equal-length kernels
    (which share the per-day sorted extremes between all replacements) but exact and copy-free."""
    import torch
    from .calendar import year_ordinals
    ta_b = ta.isel(sl)
    xb = x2d[sl.start:sl.stop]
    yidx, years = year_ordinals(ta_b)
    n_doy = int(ta_b.doy.max())
    Tb, C = xb.shape
    P = len(poff) - 1
    N = len(starts)
    acc = torch.zeros((P, C), dtype=torch.float64 if fraction else torch.int64, device=x2d.device)
    nrep = torch.zeros((P, C), dtype=torch.int64, device=x2d.device)
    ident = np.arange(Tb, dtype=np.int32)
    if blocks is None:
        blocks = []
        for yi in range(N):
            periods = np.unique(step_period[int(starts[yi]):int(starts[yi]) + int(lens[yi])])
            blocks.append((yi, int(periods[0]), int(periods[-1]) + 1))   # periods of the studied axis in block y
    for yi, p0, p1 in blocks:
        a, n = int(starts[yi]), int(lens[yi])
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
            if getattr(index, "takes_p0", False):
                v = index(xs, sub_off, doy_idx, table, p0)
            else:
                v = index(xs, sub_off, doy_idx, table)
            if fraction:
                ok = ~torch.isnan(v)
                acc[p0:p1] += torch.where(ok, v.to(torch.float64), torch.zeros_like(acc[p0:p1]))
                nrep[p0:p1] += ok.to(torch.int64)
            else:
                acc[p0:p1] += v.to(torch.int64)
                nrep[p0:p1] += 1
    if fraction:
        return torch.where(nrep > 0, acc / nrep.clamp(min=1).to(torch.float64),
                           torch.full_like(acc, float("nan"))).to(torch.float32)
    return acc.to(torch.float64) / nrep.clamp(min=1).to(torch.float64)
