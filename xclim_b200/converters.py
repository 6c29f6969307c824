"""CUDA implementation behind ``xclim.indices.converters.potential_evapotranspiration`` and ``water_budget``.

The reference evaluates the PET formulas with xarray arithmetic over the whole grid (indices/converters.py
:1890-2152) and recomputes the solar terms (indices/helpers.py:95-525) for every grid cell.  Here the solar terms
are tabulated once per (day, distinct latitude) on the host, in float64 with the reference's numpy expressions,
and one kernel pass turns the daily inputs into PET -- or straight into the water budget ``pr - PET``
(:2652-2739) without materialising PET -- in kg m-2 s-1.  The monthly methods (TW48, DA02) take daily inputs and
give one value per calendar month (``MS``).
"""
from __future__ import annotations

import warnings

import numpy as np

from . import _lib, device
from .field import Field, is_xarray, wrap_like
from .fire import _affine, _label_per_cell, _per_cell
from .generic import _unwrap, _wrap_periods
from .options import OPTIONS
from .timeaxis import _is_leap
from .units import units_of

#: method names and aliases of the reference (:2000-2147) -> kernel method
METHODS = {"baierrobertson65": "BR65", "BR65": "BR65", "hargreaves85": "HG85", "HG85": "HG85",
           "mcguinnessbordne05": "MB05", "MB05": "MB05", "allen98": "allen98", "FAO_PM98": "allen98",
           "thornthwaite48": "TW48", "TW48": "TW48", "droogersallen02": "DA02", "DA02": "DA02"}
#: unit every input is converted to, per method (the reference's convert_units_to calls)
_TARGET = {"BR65": "degF", "HG85": "degC", "MB05": "degC", "allen98": "degC", "TW48": "degC", "DA02": "degC"}
_OTHER_TARGETS = {"hurs": "", "rsds": "W m-2", "rsus": "W m-2", "rlds": "W m-2", "rlus": "W m-2",
                  "sfcWind": "m s-1", "evspsblpot": "kg m-2 s-1"}
_OUT_UNITS = "kg m-2 s-1"


# ------------------------------------------------------------------------------------ solar terms (host)
def _wrap_radians(x):
    return ((x + np.pi) % (2 * np.pi)) - np.pi


def day_angle(year, doy, calendar):
    """``helpers.day_angle`` (:95-116) of days at 00:00: the fractional part of xarray's ``dt.decimal_year``,
    ``year + (doy - 1) / days_in_year``, as an angle."""
    year = np.asarray(year, dtype=np.int64)
    if calendar == "360_day":
        n = np.full(year.shape, 360.0)
    else:
        n = np.where(_is_leap(year, calendar), 366.0, 365.0)
    decimal_year = year + (np.asarray(doy, dtype=np.float64) - 1) / n
    return (decimal_year % 1) * 2 * np.pi


def solar_declination(da):
    """Spencer's declination (:119-163), wrapped to [-pi, pi)."""
    sd = (0.006918 - 0.399912 * np.cos(da) + 0.070257 * np.sin(da) - 0.006758 * np.cos(2 * da)
          + 0.000907 * np.sin(2 * da) - 0.002697 * np.cos(3 * da) + 0.001480 * np.sin(3 * da))
    return _wrap_radians(sd)


def eccentricity_correction_factor(da):
    """Spencer's eccentricity correction (:195-238)."""
    return (1.0001100 + 0.034221 * np.cos(da) + 0.001280 * np.sin(da) + 0.000719 * np.cos(2 * da)
            + 0.000077 * np.sin(2 * da))


def _sunlit_integral_daily(decl, lat):
    """The daily branch of ``_sunlit_integral_of_cosine_of_solar_zenith_angle`` (:353-397) with h_start = -pi,
    h_end = pi - 1e-9 (:309-311) and the sunset hour angle of :332-335; ``decl`` and ``lat`` in wrapped radians."""
    h_s = _wrap_radians(-np.pi)
    h_e = _wrap_radians(np.pi - 1e-9)
    with np.errstate(invalid="ignore"):
        tantan = -np.tan(lat) * np.tan(decl)
        h_ss = _wrap_radians(np.arccos(np.where(np.abs(tantan) <= 1, tantan, np.nan)))
    h_sr = -h_ss
    polar = np.isnan(h_ss)
    day = polar & (decl * lat > 0)
    night = polar & (decl * lat < 0)
    dark = ((h_s > h_ss) & (h_e < h_sr)) | ((h_s < h_sr) & (h_e < h_sr)) | ((h_s > h_ss) & (h_e > h_ss))
    h1 = np.where(h_s > h_sr, h_s, h_sr)          # max(h_sunrise, h_start)
    h2 = np.where(h_e < h_ss, h_e, h_ss)          # min(h_sunset, h_end)
    num = np.where(day, np.sin(h_e) - np.sin(h_s), np.sin(h2) - np.sin(h1))
    denum = np.where(day, h_e - h_s, h2 - h1)
    out = np.sin(decl) * np.sin(lat) * denum + np.cos(decl) * np.cos(lat) * num
    return np.where(night | (~polar & dark), 0.0, out)


def extraterrestrial_solar_radiation(da, lat_deg, solar_constant=1361.0):
    """(:400-447) in J m-2 d-1 for day angles ``da`` (T, 1) and latitudes in degrees (1, L)."""
    lat = _wrap_radians(np.asarray(lat_deg, dtype=np.float64) * (np.pi / 180))
    gsc = solar_constant * 86400.0
    return gsc * (1 / (2 * np.pi)) * _sunlit_integral_daily(solar_declination(da), lat) * \
        eccentricity_correction_factor(da)


def day_lengths(da, lat_deg):
    """(:450-525) in hours; NaN in polar days and nights (``infill_polar_days=False``)."""
    with np.errstate(invalid="ignore"):
        return (24 / np.pi) * np.arccos(-np.tan(np.asarray(lat_deg, dtype=np.float64) * (np.pi / 180))
                                        * np.tan(solar_declination(da)))


def _daily_table(method, ta, lat_u):
    """(T, L) float64 solar term of a daily method, in the unit its formula takes."""
    da = day_angle(ta.year, ta.doy, ta.calendar)[:, None]
    if method == "BR65":
        return extraterrestrial_solar_radiation(da, lat_u[None, :]) * (1 / 41840.0)     # cal cm-2 d-1
    if method == "HG85":
        return extraterrestrial_solar_radiation(da, lat_u[None, :]) * 1e-6 * 0.408     # MJ m-2 d-1
    return extraterrestrial_solar_radiation(da, lat_u[None, :], 1367.0)                 # MB05, J m-2 d-1


def _month_days(year, month, calendar):
    if calendar == "360_day":
        return 30
    dpm = [31, 29 if bool(_is_leap(np.array(year), calendar)) else 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31]
    return dpm[month - 1]


def _months(ta):
    """Row offsets (M + 1), YS-group month offsets (Y + 1), (year, month) and length of every calendar month the
    series touches."""
    poff = ta.period_offsets("MS")
    ym = [(int(ta.year[i]), int(ta.month[i])) for i in poff[:-1]]
    years = np.array([y for y, _ in ym])
    cuts = np.nonzero(np.diff(years) != 0)[0] + 1
    yoff = np.concatenate([[0], cuts, [len(ym)]]).astype(np.int32)
    mdays = np.array([_month_days(y, m, ta.calendar) for y, m in ym], dtype=np.float64)
    return poff.astype(np.int32), yoff, ym, mdays


def _monthly_table(method, ta, ym, lat_u):
    """(M, L) float64: the mean day length / 12 (TW48) or 0.408 * the radiation sum in MJ m-2 d-1 (DA02) over each
    COMPLETE calendar month (``_get_D_from_M``, :1798-1812), skipna like xarray's resample."""
    rows = []
    for y, m in ym:
        n = _month_days(y, m, ta.calendar)
        start = 1 + (30 * (m - 1) if ta.calendar == "360_day" else
                     sum(_month_days(y, k, ta.calendar) for k in range(1, m)))
        da = day_angle(np.full(n, y), np.arange(start, start + n), ta.calendar)[:, None]
        with np.errstate(invalid="ignore"), warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)     # polar months: the mean of no day length is NaN
            if method == "TW48":
                rows.append(np.nanmean(day_lengths(da, lat_u[None, :]) / 12, axis=0))
            else:
                rows.append(np.nansum(extraterrestrial_solar_radiation(da, lat_u[None, :]) * 1e-6, axis=0) * 0.408)
    return np.stack(rows)


# ------------------------------------------------------------------------------------ host layer
def _gather_lat(da, func):
    """``helpers._gather_lat`` (:852-872): the latitude coordinate of ``da``."""
    coords = getattr(da, "coords", {})
    if "lat" in coords:
        c = coords["lat"]
        if is_xarray(da):
            return c
        return Field(np.asarray(c.values if hasattr(c, "values") else c), ("lat",), None, {}, {})
    raise ValueError(f"{func} could not find latitude coordinate in DataArray. Try passing it explicitly "
                     "(`lat=ds.lat`).")


def _check_daily(ta):
    """The series must be daily without gaps: every day follows the previous one in its calendar."""
    if len(ta) < 2:
        return
    y = ta.year[:-1]
    if ta.calendar == "360_day":
        ylen = np.full(y.shape, 360)
    else:
        ylen = np.where(_is_leap(y, ta.calendar), 366, 365)
    last = ta.doy[:-1] == ylen
    ok = np.where(last, (ta.doy[1:] == 1) & (ta.year[1:] == y + 1), (ta.doy[1:] == ta.doy[:-1] + 1)
                  & (ta.year[1:] == y))
    if not ok.all():
        raise NotImplementedError("potential_evapotranspiration takes daily series without gaps (other "
                                  "frequencies are not supported)")


def _lat_index(lat, other, cell_shape):
    vals = _per_cell(lat, other, cell_shape, np.float64, "lat")
    lat_u, idx = np.unique(vals, return_inverse=True)
    return lat_u, idx.astype(np.int32).reshape(-1)


def _pet(*, method, lat=None, water_budget=False, **series):
    """One kernel pass over the daily series (``series``: input name -> labelled array or None)."""
    kind = METHODS.get(method, method)
    given = {k: v for k, v in series.items() if v is not None}
    template = next(iter(given.values()))
    x = {}
    cell_shape = other = ta = None
    for k, da in given.items():
        x2d, cs, od, t = _unwrap(da)
        if cell_shape is None:
            cell_shape, other, ta = cs, od, t
        elif cs != cell_shape or x2d.shape[0] != len(ta):
            raise ValueError("the input series must share their shape")
        x[k] = x2d
    _check_daily(ta)
    P = _lib.PetParams()
    P.method = _lib.PET_METHODS[kind]
    P.water_budget = int(bool(water_budget))
    for i, name in enumerate(_lib.PET_INPUTS):
        if name not in x:
            P.in_scale[i], P.in_offset[i] = 1.0, 0.0
            continue
        if name in ("tasmin", "tasmax", "tas"):
            target = _TARGET[kind]
        elif name == "pr":
            target = "mm/month" if kind == "DA02" else _OUT_UNITS
        else:
            target = _OTHER_TARGETS[name]
        P.in_scale[i], P.in_offset[i] = _affine_to(given[name], target)
    return template, x, cell_shape, other, ta, P, kind


def _affine_to(da, target):
    if target == "":
        u = units_of(da).strip()
        if u in ("%", "percent", "pct"):
            return (0.01, 0.0)
        if u in ("", "1"):
            return (1.0, 0.0)
        raise ValueError(f"Cannot convert {u!r} to '1'")
    return _affine(da, target)


def _compute(method, lat, water_budget, peta, petb, **series):
    template, x, cell_shape, other, ta, P, kind = _pet(method=method, water_budget=water_budget, **series)
    P.peta, P.petb = float(peta), float(petb)
    P.wind_num, P.wind_den = float(np.log(67.8 * 2.0 - 5.42)), float(np.log(67.8 * 10.0 - 5.42))
    dev = next(iter(x.values())).device
    inputs = [x.get(name) for name in _lib.PET_INPUTS]
    table_d = idx_d = None
    if kind not in ("allen98", "given"):
        lat_u, idx = _lat_index(lat, other, cell_shape)
        idx_d = _to_dev(idx, dev)
    attrs = {"units": _OUT_UNITS}
    if kind in _lib.PET_MONTHLY:
        moff, yoff, ym, mdays = _months(ta)
        table_d = _to_dev(_monthly_table(kind, ta, ym, lat_u), dev)
        out = device.pet_monthly(inputs, moff, yoff, mdays, table_d, idx_d, P)
        return _wrap_periods(template, out, cell_shape, other, ta, "MS", attrs)
    if table_d is None and idx_d is not None:
        table_d = _to_dev(_daily_table(kind, ta, lat_u), dev)
    out = device.pet_daily(inputs, table_d, idx_d, P)
    vals = out.reshape((out.shape[0],) + cell_shape) if out.is_contiguous() else \
        out.contiguous().reshape((out.shape[0],) + cell_shape)
    keep_dev = OPTIONS["device_outputs"] and not is_xarray(template)
    vals = vals if keep_dev else vals.cpu().numpy()
    time = ta if ta.coord is None else ta.coord
    return wrap_like(template, vals, ("time",) + tuple(other), time=time, attrs=attrs)


def _to_dev(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _prepare(method, tasmin, tasmax, tas, lat, hurs, rsds, rsus, rlds, rlus, sfcWind, pr, func):
    """Method resolution, the reference's checks and the per-method inputs."""
    if method not in METHODS:
        raise NotImplementedError(f"'{method}' method is not implemented.")
    kind = METHODS[method]
    if kind == "allen98" and sfcWind is None:
        raise ValueError("Wind speed is required for Allen98 method.")
    required = {"BR65": ("tasmin", "tasmax"), "HG85": ("tasmin", "tasmax"), "DA02": ("tasmin", "tasmax", "pr"),
                "allen98": ("tasmin", "tasmax", "hurs", "rsds", "rsus", "rlds", "rlus", "sfcWind"),
                "MB05": ("tas",) if tas is not None else ("tasmin", "tasmax"),
                "TW48": ("tas",) if tas is not None else ("tasmin", "tasmax")}[kind]
    given = dict(tasmin=tasmin, tasmax=tasmax, tas=tas, hurs=hurs, rsds=rsds, rsus=rsus, rlds=rlds, rlus=rlus,
                 sfcWind=sfcWind, pr=pr)
    for name in required:
        if given[name] is None:
            raise ValueError(f"potential_evapotranspiration(method={method!r}) needs `{name}`")
    used = {k: (v if k in required or (k == "tas" and kind in ("HG85", "DA02")) else None) for k, v in given.items()}
    if kind != "allen98" and lat is None:
        lat = _gather_lat(tasmin if tas is None else tas, func)
    if kind != "allen98":
        ref = next(v for v in used.values() if v is not None)
        lat = _label_per_cell(lat, ref)
    return kind, used, lat


def potential_evapotranspiration(tasmin=None, tasmax=None, tas=None, lat=None, hurs=None, rsds=None, rsus=None,
                                 rlds=None, rlus=None, sfcWind=None, pr=None, method="BR65",
                                 peta=0.00516409319477, petb=0.0874972822289):
    """Potential evapotranspiration [kg m-2 s-1] -- indices/converters.py:1890-2152, from daily inputs.

    BR65, HG85, MB05 and allen98 give daily values; TW48 and DA02 give one value per calendar month (``MS``), each
    month's amount divided by its length in the calendar.  Outputs are float32 (DESIGN.md section 4).
    """
    from .streaming import streamed
    kind, used, lat = _prepare(method, tasmin, tasmax, tas, lat, hurs, rsds, rsus, rlds, rlus, sfcWind, pr,
                               "potential_evapotranspiration")
    return streamed(_compute)(method, lat, False, peta, petb, **used)


def water_budget(pr, evspsblpot=None, tasmin=None, tasmax=None, tas=None, lat=None, hurs=None, rsds=None,
                 rsus=None, rlds=None, rlus=None, sfcWind=None, method="BR65"):
    """Precipitation minus potential evapotranspiration [kg m-2 s-1] -- indices/converters.py:2652-2739.

    The PET of ``method`` is computed in the same kernel pass and never stored; with ``evspsblpot`` the result is
    the plain difference.  For TW48 ``pr`` is first averaged over each calendar month (:2734-2735).
    """
    from .streaming import streamed
    if evspsblpot is not None:
        _affine(pr, _OUT_UNITS)
        return streamed(_compute)("given", None, True, 0.0, 0.0, pr=pr, evspsblpot=evspsblpot)
    if method in METHODS and METHODS[method] == "DA02":
        raise ValueError("water_budget(method='DA02') is not supported: the reference does not pass `pr` on to "
                         "potential_evapotranspiration, which needs it for DA02.")
    if lat is None:              # :2714-2715, for every method (allen98 does not use it)
        lat = _gather_lat(pr, "water_budget")
    kind, used, lat = _prepare(method, tasmin, tasmax, tas, lat, hurs, rsds, rsus, rlds, rlus, sfcWind, None,
                               "water_budget")
    used["pr"] = pr
    return streamed(_compute)(method, lat, True, 0.0, 0.0, **used)
