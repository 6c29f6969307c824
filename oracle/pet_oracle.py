"""Oracle for potential evapotranspiration and the water budget (indices/converters.py:1890-2152, 2652-2739).

A plain numpy restatement, element by element, of the solar helpers (indices/helpers.py:95-525, the sunlit
integral evaluated day by day with Python's math module), of every PET method on daily inputs, of the monthly
grouping of TW48 / DA02 and of ``amount2rate``.  Two arithmetic modes:

* ``mode="f64"`` -- the kernel contract: inputs converted in float32, every formula in float64, one rounding;
* ``mode="ref"`` -- the reference's dtypes: the temperature chains in float32 until the float64 radiation term
  enters (BR65, HG85, MB05), allen98's float32 chain, the result in float64.

Inputs are (T, C) arrays already in the units each formula takes (degF for BR65, degC otherwise, hurs as a
fraction, radiation in W m-2, wind in m s-1, pr in kg m-2 s-1 or mm/month for DA02).
"""
from __future__ import annotations

import math

import numpy as np

SOLAR_CONSTANT = 1361.0


def _leap(y, calendar):
    if calendar in ("noleap", "365_day", "360_day"):
        return False
    if calendar in ("all_leap", "366_day"):
        return True
    if calendar == "julian":
        return y % 4 == 0
    return y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)


def year_length(y, calendar):
    return 360 if calendar == "360_day" else (366 if _leap(y, calendar) else 365)


def month_lengths(y, calendar):
    if calendar == "360_day":
        return [30] * 12
    return [31, 29 if _leap(y, calendar) else 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31]


def wrap(x):
    return ((x + math.pi) % (2 * math.pi)) - math.pi


def day_angle(year, doy, calendar):
    return ((year + (doy - 1) / year_length(year, calendar)) % 1) * 2 * math.pi


def declination(da):
    return wrap(0.006918 - 0.399912 * math.cos(da) + 0.070257 * math.sin(da) - 0.006758 * math.cos(2 * da)
                + 0.000907 * math.sin(2 * da) - 0.002697 * math.cos(3 * da) + 0.001480 * math.sin(3 * da))


def eccentricity(da):
    return (1.0001100 + 0.034221 * math.cos(da) + 0.001280 * math.sin(da) + 0.000719 * math.cos(2 * da)
            + 0.000077 * math.sin(2 * da))


def sunlit_integral(decl, lat, h_ss, h_s, h_e):
    """Integral of the cosine of the solar zenith angle over the sunlit part of [h_s, h_e] (helpers.py:353-397,
    ``average=False``)."""
    h_sr = -h_ss
    if math.isnan(h_ss) and decl * lat > 0:
        num = math.sin(h_e) - math.sin(h_s)
        den = h_e + 2 * math.pi - h_s if h_e < h_s else h_e - h_s
    elif math.isnan(h_ss) and decl * lat < 0:
        return 0.0
    elif (h_s > h_ss and h_e < h_sr) or (h_s < h_sr and h_e < h_sr) or (h_s > h_ss and h_e > h_ss):
        return 0.0
    elif h_s > h_e >= h_sr and h_s >= h_ss:
        num, den = math.sin(h_e) - math.sin(h_sr), h_e - h_sr
    elif h_e < h_s and h_s >= h_sr >= h_e:
        num, den = math.sin(h_ss) - math.sin(h_s), h_ss - h_s
    elif h_ss >= h_s > h_e >= h_sr:
        num = math.sin(h_ss) - math.sin(h_s) + math.sin(h_e) - math.sin(h_sr)
        den = h_ss - h_s + h_e - h_sr
    else:
        h1, h2 = max(h_sr, h_s), min(h_ss, h_e)
        num, den = math.sin(h2) - math.sin(h1), h2 - h1
    return math.sin(decl) * math.sin(lat) * den + math.cos(decl) * math.cos(lat) * num


def radiation(year, doy, calendar, lat_deg, solar_constant=SOLAR_CONSTANT):
    """Daily extraterrestrial radiation [J m-2 d-1] (helpers.py:400-447)."""
    da = day_angle(year, doy, calendar)
    decl = declination(da)
    lat = wrap(lat_deg * (math.pi / 180))
    tt = -math.tan(lat) * math.tan(decl)
    h_ss = wrap(math.acos(tt)) if abs(tt) <= 1 else math.nan
    integral = sunlit_integral(decl, lat, h_ss, wrap(-math.pi), wrap(math.pi - 1e-9))
    return solar_constant * 86400.0 * (1 / (2 * math.pi)) * integral * eccentricity(da)


def day_length(year, doy, calendar, lat_deg):
    """Day length [h] (helpers.py:450-525), NaN in polar days and nights."""
    tt = -math.tan(lat_deg * (math.pi / 180)) * math.tan(declination(day_angle(year, doy, calendar)))
    return (24 / math.pi) * math.acos(tt) if abs(tt) <= 1 else math.nan


def radiation_table(years, doys, calendar, lats, solar_constant=SOLAR_CONSTANT):
    return np.array([[radiation(int(y), int(d), calendar, float(la), solar_constant) for la in lats]
                     for y, d in zip(years, doys)])


# ------------------------------------------------------------------------------------ daily methods
def esat(tk):
    return 100 * np.exp(-6096.9385 / tk + 16.635794 + -2.711193e-2 * tk + 1.673952e-5 * tk ** 2 + 2.433502 * np.log(tk))


def _clip0(v):
    return np.where(v < 0, 0.0, v)


def daily_pet(method, rad, tasmin=None, tasmax=None, tas=None, hurs=None, rsds=None, rsus=None, rlds=None,
              rlus=None, sfcWind=None, peta=0.00516409319477, petb=0.0874972822289, mode="f64"):
    """PET [mm/d] of a daily method; ``rad`` (T, C): the method's radiation term (cal cm-2 d-1 for BR65,
    0.408 * MJ m-2 d-1 for HG85, J m-2 d-1 with 1367 W m-2 for MB05; unused for allen98)."""
    f = np.float64 if mode == "f64" else np.float32

    def a(x):
        return None if x is None else np.asarray(x, dtype=np.float32).astype(f)

    tn, tx, tm = a(tasmin), a(tasmax), a(tas)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        if method == "BR65":
            return _clip0(0.094 * (-87.03 + 0.928 * tx + 0.933 * (tx - tn) + 0.0486 * rad))
        if method == "HG85":
            t = (tn + tx) / 2 if tm is None else tm
            return _clip0(0.0023 * rad * (t + 17.8) * (tx - tn) ** 0.5)
        if method == "MB05":
            t = (tn + tx) / 2 if tm is None else tm
            tk = t + f(273.15) if mode == "ref" else t + 273.15
            r = rad / (4185.5 * (751.78 - 0.5655 * tk))
            return r * peta * t + r * petb
        if method == "allen98":
            u2 = a(sfcWind) * math.log(67.8 * 2 - 5.42) / math.log(67.8 * 10 - 5.42)
            t = (tx + tn) / 2
            es = 0.5 * (esat(tx + 273.15) + esat(tn + 273.15)) / 1000
            ea = es * a(hurs)
            delta = 4098 * es / (t + 237.3) ** 2
            rn = (a(rsds) - a(rsus) - (a(rlus) - a(rlds))) * 0.0864
            gamma = 0.665e-03 * 101.325
            a1 = 0.408 * delta * (rn - 0)
            a2 = gamma * 900 / (t + 273.15) * u2 * (es - ea)
            a3 = delta + gamma * (1 + 0.34 * u2)
            return (a1 + a2) / a3
    raise NotImplementedError(method)


def daily_rate(pet_mm, pr=None):
    """amount2rate over one day and mm/d -> kg m-2 s-1; minus the water budget's pr when given."""
    rate = np.asarray(pet_mm, dtype=np.float64) / 1.0 / 86400.0
    return rate if pr is None else np.asarray(pr, dtype=np.float32).astype(np.float64) - rate


# ------------------------------------------------------------------------------------ monthly methods
def months(years, mons):
    """[(year, month, first row, end row)] of the calendar months a daily series touches, in order."""
    out = []
    for i, (y, m) in enumerate(zip(years, mons)):
        if not out or tuple(out[-1][:2]) != (int(y), int(m)):
            out.append([int(y), int(m), i, i + 1])
        else:
            out[-1][3] = i + 1
    return [tuple(v) for v in out]


def _month_doys(y, m, calendar):
    ml = month_lengths(y, calendar)
    start = 1 + sum(ml[:m - 1])
    return range(start, start + ml[m - 1])


def _nanmean(x):
    n = (~np.isnan(x)).sum(0)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(n > 0, np.nansum(x, 0) / n, np.nan)


def monthly_pet(method, years, mons, doys, calendar, lats, tasmin=None, tasmax=None, tas=None, pr=None, wb_pr=None):
    """(M, C) TW48 / DA02 rate [kg m-2 s-1] from daily (T, C) inputs, or the water budget with ``wb_pr``
    (kg m-2 s-1) when given; ``lats`` (C,) degrees."""
    f = np.float64
    tn = None if tasmin is None else np.asarray(tasmin, np.float32).astype(f)
    tx = None if tasmax is None else np.asarray(tasmax, np.float32).astype(f)
    tm = (tn + tx) / 2 if tas is None else np.asarray(tas, np.float32).astype(f)
    ms = months(years, mons)
    lat_u = np.asarray(lats, dtype=np.float64)
    out = np.empty((len(ms), tm.shape[1]))
    with np.errstate(invalid="ignore", divide="ignore"):
        if method == "DA02":
            prm = np.asarray(pr, np.float32).astype(f)
            for k, (y, m, a, b) in enumerate(ms):
                ra = np.array([np.nansum([radiation(y, d, calendar, la) * 1e-6 for d in _month_doys(y, m, calendar)])
                               for la in lat_u]) * 0.408
                tr = _nanmean(tx[a:b]) - _nanmean(tn[a:b])
                tr = np.where(tr > 0, tr, 0)
                ab = tr - 0.0123 * _nanmean(prm[a:b])
                p = ab ** 0.76
                pet = _clip0(np.where(np.isnan(p), 0, 0.0013 * ra * (_nanmean(tm[a:b]) + 17.0) * p))
                out[k] = pet / month_lengths(y, calendar)[m - 1] / 86400.0
            return out
        tmc = np.where(tm < 0, 0.0, tm)
        tmean = np.stack([_nanmean(tmc[a:b]) for (_, _, a, b) in ms])
        prm = None if wb_pr is None else np.stack([_nanmean(np.asarray(wb_pr, np.float32).astype(f)[a:b])
                                                   for (_, _, a, b) in ms])
        years_m = np.array([y for (y, _, _, _) in ms])
        for y in np.unique(years_m):
            sel = np.nonzero(years_m == y)[0]
            i_m = (tmean[sel] / 5) ** 1.514
            heat = np.nansum(i_m, axis=0)
            a_ = 6.75e-7 * heat ** 3 - 7.71e-5 * heat ** 2 + 0.01791 * heat + 0.49239
            for k in sel:
                yy, m = ms[k][:2]
                dl = np.array([np.nanmean([day_length(yy, d, calendar, la) / 12 for d in _month_doys(yy, m, calendar)])
                               for la in lat_u])
                pet = 10 * (1.6 * dl * (10 * tmean[k] / heat) ** a_)
                out[k] = pet / month_lengths(yy, calendar)[m - 1] / 86400.0
                if prm is not None:
                    out[k] = prm[k] - out[k]
    return out
