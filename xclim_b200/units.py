"""Scalar unit handling on the host (only what reaches the kernels: one threshold value).

The reference uses pint/cf_xarray (core/units.py:334-451 `convert_units_to`, 621-741
`to_agg_units`); none of that is array math.  When the real xclim is importable its
``convert_units_to`` is used; otherwise a small table covers the units of the hot-path configs.
"""
from __future__ import annotations

import re

try:  # pragma: no cover - only where the reference is installed
    from xclim.core.units import convert_units_to as _xclim_convert  # type: ignore
except Exception:
    _xclim_convert = None

_ALIASES = {
    "k": "K", "kelvin": "K", "degk": "K",
    "degc": "degC", "°c": "degC", "c": "degC", "celsius": "degC", "deg_c": "degC",
    "degf": "degF", "°f": "degF",
    "mm/d": "mm/d", "mm/day": "mm/d", "mm d-1": "mm/d", "mm day-1": "mm/d", "mm d^-1": "mm/d",
    "kg m-2 s-1": "kg m-2 s-1", "kg/m2/s": "kg m-2 s-1", "kg m^-2 s^-1": "kg m-2 s-1", "mm/s": "kg m-2 s-1",
    "mm": "mm", "d": "d", "days": "d", "day": "d", "": "", "1": "", "m/s": "m s-1", "m s-1": "m s-1",
    "km h-1": "km h-1", "km/h": "km h-1", "kph": "km h-1", "km hr-1": "km h-1",
    "kg/m**2/s": "kg m-2 s-1", "kg m**-2 s**-1": "kg m-2 s-1",
    "%": "%", "percent": "%", "pct": "%",
    "w m-2": "W m-2", "w/m2": "W m-2", "w m^-2": "W m-2", "w m**-2": "W m-2", "w/m^2": "W m-2", "w/m**2": "W m-2",
    "mm/month": "mm/month", "mm month-1": "mm/month",
}
#: pint's default registry: month = year / 12, year = 365.25 d
_DAYS_PER_MONTH = 365.25 / 12


def _canon(u: str) -> str:
    key = u.strip().lower()
    return _ALIASES.get(key, u.strip())


def parse_quantity(q):
    """"1 mm/day" -> (1.0, "mm/day"); numbers pass through with units None."""
    if isinstance(q, (int, float)):
        return float(q), None
    # 1, 1.5, .5, 10., 1e-5, 1E6 (what Python's float() accepts, without inf / nan)
    m = re.fullmatch(r"\s*([-+]?(?:[0-9]+\.?[0-9]*|\.[0-9]+)(?:[eE][-+]?[0-9]+)?)\s*(.*)", str(q))
    if not m:
        raise ValueError(f"Cannot parse quantity {q!r}")
    return float(m.group(1)), m.group(2).strip()


def _to_base(v: float, u: str):
    if u == "K":
        return v, "temp"
    if u == "degC":
        return v + 273.15, "temp"
    if u == "degF":
        return (v - 32.0) * 5.0 / 9.0 + 273.15, "temp"
    if u == "mm/d":
        return v / 86400.0, "prflux"
    if u == "kg m-2 s-1":
        return v, "prflux"
    if u == "mm/month":
        return v / (86400.0 * _DAYS_PER_MONTH), "prflux"
    if u == "%":
        return v / 100.0, "ratio"
    if u == "":
        return v, "ratio"
    if u == "W m-2":
        return v, "radflux"
    if u == "m s-1":
        return v, "speed"
    if u == "km h-1":
        return v / 3.6, "speed"
    return v, u


def _from_base(v: float, u: str):
    if u == "K":
        return v
    if u == "degC":
        return v - 273.15
    if u == "degF":
        return (v - 273.15) * 9.0 / 5.0 + 32.0
    if u == "mm/d":
        return v * 86400.0
    if u == "km h-1":
        return v * 3.6
    if u == "mm/month":
        return v * (86400.0 * _DAYS_PER_MONTH)
    if u == "%":
        return v * 100.0
    return v


def convert_units_to(source, target_units: str, context=None) -> float:
    """Threshold (str | number) expressed in ``target_units`` as a Python float
    (core/units.py:398-403: a string source yields ``float``)."""
    val, u = parse_quantity(source)
    if u is None:
        return val
    cu, ct = _canon(u), _canon(target_units)
    if cu == ct:
        return val
    base, kind = _to_base(val, cu)
    _, kind_t = _to_base(0.0, ct)
    if kind != kind_t or kind in (cu,):
        raise ValueError(f"Cannot convert {u!r} to {target_units!r} (install xclim for full pint support)")
    return float(_from_base(base, ct))


def units_of(da) -> str:
    u = da.attrs.get("units")
    if u is None:
        raise ValueError("input has no `units` attribute")
    return u


def threshold_in_units_of(thresh, da) -> float:
    """``convert_units_to(thresh, da, context="infer")`` -> Python float."""
    if _xclim_convert is not None and hasattr(da, "coords"):
        try:  # pragma: no cover
            return float(_xclim_convert(thresh, da, context="infer"))
        except Exception:
            pass
    return convert_units_to(thresh, units_of(da))


def to_agg_units_attrs(da, op: str) -> dict:
    """The ``units`` attr the reference's ``to_agg_units`` sets (core/units.py:621-741) for DAILY
    data: count-like ops -> "d" (x1 day per step, :704-712); mean/min/max/sum(integral aside)
    keep the input units (:696-697); std keeps units, var squares them."""
    u = da.attrs.get("units", "")
    if op in ("count", "doymin", "doymax"):
        return {"units": "d"}
    if op == "var":
        return {"units": f"({u})^2" if u else ""}
    return {"units": u}
