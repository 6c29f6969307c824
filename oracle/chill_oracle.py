"""Numpy restatement of the chill indices, step by step, for the tests.

- ``hourly_temperature``: ``make_hourly_temperature`` (indices/helpers.py:1059-1123) with the day lengths given:
  the daily values repeated 24 times (``resample("h").ffill()``), the next day's tasmin (``shift(time=-1)`` after
  a copy of the last day), then ``xr.where(hour < dl, day, night)`` with the reference's expressions, in its dtype
  promotion (``tasmax - tasmin`` in the input dtype).
- ``dynamic``: ``_chill_portion_one_season`` (indices/_agro.py:1436-1465) on one period, hour loop in float64.
- ``utah``: the weights of ``chill_units`` (:1537-1592), NaN where the hour is NaN.
- ``chill``: both per period over an hourly (H, C) series, with a per-day selection (skipped days).
"""
from __future__ import annotations

import numpy as np

E0, E1, A0, A1, SLP, TETMLT = 4153.5, 12888.8, 139500, 2.567e18, 1.6, 277
AA, EE = A0 / A1, E1 - E0


def hourly_temperature(tasmin, tasmax, dl):
    """(24 T, C) float64 from daily (T, C) ``tasmin`` / ``tasmax`` and day lengths ``dl`` (T, C) in hours."""
    T = tasmin.shape[0]
    nxt = np.concatenate([tasmin[1:], tasmin[-1:]])
    rep = lambda a: np.repeat(a, 24, axis=0)  # noqa: E731
    hour = np.tile(np.arange(24, dtype=np.int64), T)[:, None]
    mn, mx, n, d = rep(tasmin), rep(tasmax), rep(nxt), rep(dl)
    with np.errstate(invalid="ignore", divide="ignore"):
        sunset = (rep(tasmax) - rep(tasmin)) * np.sin((np.pi * d) / (d + 4)) + mn
        day = (mx - mn) * np.sin((np.pi * hour) / (d + 4)) + mn
        night_h = (hour + 1 - d).clip(1)
        dlm1 = d - 1
        night = sunset - ((sunset - n) / np.log(24 - dlm1)) * np.log(night_h)
    return np.where(hour < d, day, night)


def dynamic(tk):
    """(sum, E, delta) of one period's hours ``tk`` (n,) in K, float64, the reference's hour loop."""
    tk = np.asarray(tk, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        ftmprt = SLP * TETMLT * (tk - TETMLT) / tk
        sr = np.exp(ftmprt)
        xi = sr / (1 + sr)
        xs = AA * np.exp(EE / tk)
        ak1 = A1 * np.exp(-E1 / tk)
        E = np.zeros_like(tk)
        for i in range(1, tk.size):
            S = np.where(E[i - 1] < 1, E[i - 1], E[i - 1] - E[i - 1] * xi[i - 1])
            E[i] = xs[i] - (xs[i] - S) * np.exp(-ak1[i])
        delta = np.where(E >= 1, E * xi, 0)
    s = 0.0
    for v in delta:
        s += v
    return s, E, delta


def utah(t):
    t = np.asarray(t, np.float64)
    cu = np.where((t <= 1.4) | ((t > 12.4) & (t <= 15.9)), 0.0,
                  np.where(((t > 1.4) & (t <= 2.4)) | ((t > 9.1) & (t <= 12.4)), 0.5,
                           np.where((t > 2.4) & (t <= 9.1), 1.0, np.where((t > 15.9) & (t <= 17.9), -0.5, -1.0))))
    return np.where(np.isnan(t), np.nan, cu)


def chill(hourly, poff, mask=None, to_k=(1.0, 0.0), to_c=(1.0, -273.15), positive_only=False):
    """``(cp, cu, valid)`` float64 / int (P, C) of an hourly (H, C) series over day offsets ``poff``; days with
    ``mask`` False are skipped.  The hours are converted with ``v * scale + offset``."""
    hourly = np.asarray(hourly, np.float64)
    H, C = hourly.shape
    P = len(poff) - 1
    cp, cu, valid = np.zeros((P, C)), np.zeros((P, C)), np.zeros((P, C), np.int64)
    for p in range(P):
        days = [d for d in range(poff[p], poff[p + 1]) if mask is None or mask[d]]
        hrs = np.array([h for d in days for h in range(24 * d, min(24 * d + 24, H))], dtype=np.int64)
        for c in range(C):
            v = hourly[hrs, c]
            valid[p, c] = int(np.sum(~np.isnan(v)))
            cp[p, c] = dynamic(v * to_k[0] + to_k[1])[0]
            w = utah(v * to_c[0] + to_c[1])
            if positive_only:
                tot = 0.0
                for d in days:
                    sel = (hrs >= 24 * d) & (hrs < 24 * d + 24)
                    daily = np.nansum(w[sel])
                    tot += daily if daily > 0 else 0.0
                cu[p, c] = tot
            else:
                cu[p, c] = np.nansum(w)
    return cp, cu, valid
