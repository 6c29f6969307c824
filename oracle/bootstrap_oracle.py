"""CPU oracle for the percentile bootstrap of any day-of-year percentile index.  TEST INFRASTRUCTURE ONLY (see
xclim_oracle.py for the conventions).

``bootstrap_doy_index`` restates ``bootstrap_func`` (core/bootstrapping.py:81-211) with ``build_bootstrap_year_da``
(:235-282) literally: it walks the bootstrap year groups, applies the index to each group's own slice of the series,
and for a group whose label year is a year of the base (:184) averages the index over the tables recomputed on the
base with that group's block replaced by each other base block.
"""
from __future__ import annotations

import numpy as np

from oracle import etccdi_oracle as E
from oracle import xclim_oracle as O


def replaced_block(xb, pos_y, pos_s, feb29_y, feb29_s):
    """The base series with block y replaced by block s (core/bootstrapping.py:255-279); a copy of it unchanged
    where the reference leaves the block untouched.  ``feb29_*``: position of Feb 29 inside the block, or None."""
    z = xb.copy()
    ly, ls = len(pos_y), len(pos_s)
    if ls < 360 and ls < ly:                                      # :257-260
        return z
    if ls == ly:                                                  # :264-265
        z[pos_y] = xb[pos_s]
    elif ly == 365 and ls == 366:                                 # convert_calendar("noleap"): drop Feb 29
        z[pos_y] = np.delete(xb[pos_s], feb29_s, axis=0)
    elif ly == 366 and ls == 365:                                 # convert_calendar("366_day", missing=NaN)
        z[pos_y] = np.insert(xb[pos_s], feb29_y, np.nan, axis=0)
    elif ly < 365 and ls >= ly:                                   # :270-273
        z[pos_y] = xb[pos_s][:ly]
    else:
        raise NotImplementedError("unequal year blocks")
    return z


def fraction_mean(vals):
    """Mean of the float32 fractions over the replacements: float64 sum of the non-NaN terms in order over their
    number, rounded once to float32; NaN when every term is NaN."""
    v = np.asarray(vals, dtype=np.float32)
    out = np.full(v.shape[1:], np.nan, dtype=np.float32)
    for idx in np.ndindex(*v.shape[1:]):
        s, n = 0.0, 0
        for k in range(v.shape[0]):
            f = v[(k,) + idx]
            if f == f:
                s += float(f)
                n += 1
        if n:
            out[idx] = np.float32(s / n)
    return out


def bootstrap_doy_index(x, year, doy, gid, label, poff, base_years, index, window=5, per=90.0, alpha=1 / 3.,
                        beta=1 / 3., table=None, feb29=None, fraction=False):
    """``index(x_slice, table, doy_slice, poff_slice) -> (P_slice, ...)`` bootstrapped.  ``gid``: bootstrap year
    group of every step (xclim's ``_get_bootstrap_freq`` groups) and ``label`` its label year (the year of the
    group's start for ``YS*``, of its end for ``YE*``); ``base_years`` (first, last) calendar year of the
    climatology; ``feb29``: bool per step (leap days, for the 365 <-> 366 conversion).  Integer indices are averaged
    as numpy's mean (float64), fractions by ``fraction_mean``.  Returns ``(P, ...)``."""
    x = np.asarray(x)
    year, doy, gid, label = np.asarray(year), np.asarray(doy), np.asarray(gid), np.asarray(label)
    feb29 = np.zeros(len(x), bool) if feb29 is None else np.asarray(feb29)
    y0, y1 = base_years
    in_base = (year >= y0) & (year <= y1)
    if in_base.all():
        raise KeyError("`bootstrap` is unnecessary when all years are overlapping")
    if not in_base.any():
        raise KeyError("`bootstrap` is unnecessary when no year overlap")
    xb, yb, db, gb, fb = x[in_base], year[in_base], doy[in_base], gid[in_base], feb29[in_base]
    if table is None:
        table = O.percentile_doy(xb, yb, db, window, per, alpha, beta)[:, 0]
    bgroups = list(dict.fromkeys(gb.tolist()))
    out = []
    for g in list(dict.fromkeys(gid.tolist())):                  # the year groups in time order
        rows = np.nonzero(gid == g)[0]
        a, e = int(rows[0]), int(rows[-1]) + 1
        off = np.asarray(poff)
        sub = off[(off >= a) & (off <= e)] - a                   # the periods nest in the group
        xs, ds = x[a:e], doy[a:e]
        if int(label[a]) in set(yb.tolist()):                     # _get_year_label(year_key) in overlap years
            pos_y = np.nonzero(gb == g)[0]
            fy = np.nonzero(fb[pos_y])[0]
            vals = []
            for s in bgroups:
                if s == g:
                    continue
                pos_s = np.nonzero(gb == s)[0]
                fs = np.nonzero(fb[pos_s])[0]
                z = replaced_block(xb, pos_y, pos_s, fy[0] if fy.size else None, fs[0] if fs.size else None)
                tab = O.percentile_doy(z, yb, db, window, per, alpha, beta)[:, 0]
                vals.append(index(xs, tab, ds, sub))
            out.append(fraction_mean(vals) if fraction else
                       np.mean(np.stack(vals, axis=0).astype(np.float64), axis=0))
        else:
            v = index(xs, table, ds, sub)
            out.append(np.asarray(v, dtype=np.float32 if fraction else np.float64))
    return np.concatenate(out, axis=0)


# the index callables, as the reference applies them to one year slice
def count_index(op=">", floor=None, cal_max_doy=None):
    """doy_threshold_count against the table floored like days_over_precip_thresh (indices/_multivariate.py:1222)."""
    def f(xs, tab, ds, sub):
        if floor is not None:
            with np.errstate(invalid="ignore"):
                tab = np.where(tab > floor, tab, floor)
        return O.doy_threshold_count(xs, tab, ds, sub, op, cal_max_doy)
    return f


def spell_index(name, window=6, resample_before_rl=True, op=None, cal_max_doy=None):
    fn = getattr(E, name)
    kw = {} if op is None else {"op": op}
    return lambda xs, tab, ds, sub: fn(xs, tab, ds, sub, window, resample_before_rl, cal_max_doy=cal_max_doy, **kw)


def fraction_index(thresh, op=">", cal_max_doy=None):
    return lambda xs, tab, ds, sub: E.fraction_over_precip_thresh(xs, tab, thresh, sub, op, doy=ds,
                                                                  cal_max_doy=cal_max_doy)
