"""Generate tests/golden/ref_pet.npz: the reference's own solar helpers on every day of 360-, 365- and 366-day years.

Runs ``extraterrestrial_solar_radiation`` (with ``cosine_of_solar_zenith_angle``, ``solar_declination``,
``eccentricity_correction_factor``, ``day_angle`` and the numba ``_sunlit_integral_of_cosine_of_solar_zenith_angle``)
and ``day_lengths`` of indices/helpers.py where they lie (``_ref_extract``), and stores inputs and outputs only.
Usage: ``XCLIM_REFERENCE_ROOT=/path/to/xclim python tests/golden/make_golden_pet.py``.

xarray, pint and cftime need not be installed: the helpers run on small stand-ins.
- A float64 ndarray subclass carries ``attrs`` / ``assign_attrs`` / ``rename`` / ``where``.
- ``convert_units_to`` knows only the four conversions the helpers make: degrees_north -> rad is x * (pi / 180), as
  pint's degree; W m-2 -> J m-2 d-1 is x * 86400; "0 °" -> 0 rad; and the identities.
- ``xr.apply_ufunc`` calls the numba function on the broadcast arrays.
- ``xr.infer_freq`` answers "D", which takes the daily branch of the sunlit integral.
- The time stand-in's ``dt.decimal_year`` is xarray's definition at 00:00 (xarray >= 2024.09, ``XR2409``):
  ``year + (doy - 1) / days_in_year`` of the calendar.  That day-angle convention is the one input here that
  does not come from the reference's code.

Cases: latitudes every 10 degrees from -90 to 90 plus both polar circles (+-66.5, +-66.6, +-67), both tropics,
+-89.9 and 0; every day of year 2001 in the 360_day and noleap calendars and of year 2000 in the standard one.
"""
from __future__ import annotations

import contextlib
import os
import sys
from collections.abc import Callable, Mapping
from datetime import timedelta
from inspect import stack
from typing import Any, Literal, cast

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import _ref_extract  # noqa: E402

LATS = np.unique(np.r_[np.arange(-90.0, 91.0, 10.0), -66.5, 66.5, -66.6, 66.6, -67.0, 67.0, -23.44, 23.44, -89.9,
                       89.9, 0.0])
CASES = (("360_day", 2001, 360), ("noleap", 2001, 365), ("standard", 2000, 366))
FUNCS = ["_wrap_radians", "day_angle", "solar_declination", "eccentricity_correction_factor",
         "cosine_of_solar_zenith_angle", "_sunlit_integral_of_cosine_of_solar_zenith_angle",
         "extraterrestrial_solar_radiation", "day_lengths"]


class A(np.ndarray):
    """float64 array with the few DataArray members the helpers touch."""

    def __new__(cls, values, units=None):
        obj = np.asarray(values, dtype=np.float64).view(cls)
        obj.attrs = {} if units is None else {"units": units}
        return obj

    def __array_finalize__(self, obj):
        self.attrs = {}

    def assign_attrs(self, **kw):
        self.attrs = {**self.attrs, **kw}
        return self

    def rename(self, *_):
        return self

    def where(self, cond):
        return A(np.where(cond, self, np.nan))

    @property
    def coords(self):
        return {}


class _DT:
    def __init__(self, decimal_year, calendar):
        self.decimal_year = A(decimal_year)
        self.calendar = calendar


class Times:
    """A daily time coordinate: ``len``, ``.time`` and ``.dt.decimal_year`` (column vector, to broadcast on lat)."""

    def __init__(self, year, n, calendar):
        self.n = n
        self.dt = _DT((year + np.arange(n) / n)[:, None], calendar)

    def __len__(self):
        return self.n

    @property
    def time(self):
        return self


class _XR:
    class DataArray:
        pass

    class Dataset:
        pass

    class DataTree:
        pass

    @staticmethod
    def set_options(**_):
        return contextlib.nullcontext()

    @staticmethod
    def infer_freq(_):
        return "D"

    @staticmethod
    def apply_ufunc(func, *args, **_):
        return A(func(*[np.asarray(a) if isinstance(a, np.ndarray) else a for a in args]))


def convert_units_to(x, target, context=None):
    if isinstance(x, str):
        v, u = x.split(" ", 1)
        return {("W m-2", "J m-2 d-1"): float(v) * 86400.0, ("°", "rad"): float(v) * (np.pi / 180)}[(u, target)]
    u = x.attrs.get("units")
    if u == target or (u == "degrees_north" and target == "deg"):
        return x
    if u == "degrees_north" and target == "rad":
        return A(x * (np.pi / 180), "rad")
    raise ValueError(f"no stand-in conversion {u!r} -> {target!r}")


def load_helpers():
    import numba as nb
    ns = {"np": np, "nb": nb, "xr": _XR, "cast": cast, "Literal": Literal, "Any": Any, "Mapping": Mapping,
          "Callable": Callable, "Quantified": object, "XR2409": True, "convert_units_to": convert_units_to,
          "_chunk_like": lambda *a, chunks=None: a, "CFTimeIndex": object, "timedelta": timedelta, "stack": stack}
    return _ref_extract._extract("src/xclim/indices/helpers.py", FUNCS, ns)


def main():
    import numba
    f = load_helpers()
    lat = A(LATS[None, :], "degrees_north")
    out = {"lats": LATS, "numba_version": np.array(numba.__version__)}
    for cal, year, n in CASES:
        times = Times(year, n, cal)
        out[f"rad1361_{cal}"] = np.asarray(f["extraterrestrial_solar_radiation"](times, lat))
        out[f"rad1367_{cal}"] = np.asarray(f["extraterrestrial_solar_radiation"](times, lat, solar_constant="1367 W m-2"))
        with np.errstate(invalid="ignore"):
            out[f"daylen_{cal}"] = np.asarray(f["day_lengths"](times, lat))
        out[f"year_{cal}"] = np.array(year)
    path = os.path.join(HERE, "ref_pet.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
