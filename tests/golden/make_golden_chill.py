"""Generate tests/golden/ref_chill.npz: the reference's own hourly-temperature and chill-portion code on seeded
daily tasmin / tasmax at latitudes from -90 to 90, on a 360-, 365- and 366-day year.

Runs, where they lie (``_ref_extract``): ``day_lengths`` (with its solar helpers, as ``make_golden_pet.py`` does),
``_compute_daytime_temperature`` and ``_compute_nighttime_temperature`` of indices/helpers.py, and
``_accumulate_intermediate`` and ``_chill_portion_one_season`` of indices/_agro.py.  The xarray glue of
``make_hourly_temperature`` (indices/helpers.py:1097-1123) is restated on numpy arrays: each day's values repeated
over its 24 hours (``resample("h").ffill()``), the next day's tasmin with the last day's own at the end
(``concat`` + ``shift(time=-1)``), the hour of day, ``(hour + 1 - daylength).clip(1)`` and ``where(hour <
daylength, day, night)``.  Stores inputs and outputs only.
Usage: ``XCLIM_REFERENCE_ROOT=/path/to/xclim python tests/golden/make_golden_chill.py``.

Cases: latitudes -90, -75, -67, -66.5, -45, -23.44, 0, 30, 60, 66.6, 70, 89.9, 90; tasmin uniform in [-15, 15] degC
and tasmax = tasmin + [0, 15] (float32), NaN on a few days; day lengths with and without ``infill_polar_days``.
Hourly temperatures are stored for every 10th day (all 24 hours), chill portions (tasmin / tasmax in degC, the
hours + 273.15 in K, one season over the whole year) as the float64 sum of ``delta`` and its count of non-zero
hours.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import _ref_extract  # noqa: E402
import make_golden_pet as pet  # noqa: E402

LATS = np.array([-90.0, -75.0, -67.0, -66.5, -45.0, -23.44, 0.0, 30.0, 60.0, 66.6, 70.0, 89.9, 90.0])
CASES = pet.CASES
KEEP_EVERY = 10


class _Ufuncs:
    isnan = staticmethod(lambda x: np.isnan(np.asarray(x)))


def _where(self, cond, other=np.nan):
    return pet.A(np.where(cond, self, other))


# the two DataArray members ``day_lengths(infill_polar_days=True)`` adds to those make_golden_pet.py stands in for
pet._XR.broadcast = staticmethod(lambda *a: tuple(pet.A(v) for v in np.broadcast_arrays(*a)))
pet._XR.ufuncs = _Ufuncs
pet.A.where = _where


def load():
    h = _ref_extract._extract("src/xclim/indices/helpers.py",
                              ["_compute_daytime_temperature", "_compute_nighttime_temperature"], {"np": np})
    a = _ref_extract._extract("src/xclim/indices/_agro.py", ["_accumulate_intermediate", "_chill_portion_one_season"],
                              {"np": np})
    return h, a


def hourly(h, tasmin, tasmax, dl):
    T = tasmin.shape[0]
    nxt = np.concatenate([tasmin[1:], tasmin[-1:]])
    sunset = h["_compute_daytime_temperature"](dl, tasmin, tasmax, dl)
    rep = lambda v: np.repeat(v, 24, axis=0)  # noqa: E731
    hour = np.tile(np.arange(24, dtype=np.int64), T)[:, None]
    d = rep(dl)
    with np.errstate(invalid="ignore", divide="ignore"):
        night_h = (hour + 1 - d).clip(1)
        return np.where(hour < d, h["_compute_daytime_temperature"](hour, rep(tasmin), rep(tasmax), d),
                        h["_compute_nighttime_temperature"](night_h, rep(nxt), rep(sunset), d - 1))


def main():
    f = pet.load_helpers()
    h, a = load()
    rng = np.random.default_rng(1990)
    out = {"lats": LATS, "keep_every": np.array(KEEP_EVERY)}
    lat = pet.A(LATS[None, :], "degrees_north")
    for cal, year, n in CASES:
        times = pet.Times(year, n, cal)
        tasmin = rng.uniform(-15, 15, (n, LATS.size)).astype(np.float32)
        tasmax = (tasmin + rng.uniform(0, 15, (n, LATS.size))).astype(np.float32)
        tasmin[rng.integers(0, n, 3), rng.integers(0, LATS.size, 3)] = np.nan
        out[f"tasmin_{cal}"], out[f"tasmax_{cal}"], out[f"year_{cal}"] = tasmin, tasmax, np.array(year)
        for infill in (False, True):
            with np.errstate(invalid="ignore"):
                dl = np.asarray(f["day_lengths"](times, lat, infill_polar_days=infill))
            hr = hourly(h, tasmin, tasmax, dl)
            with np.errstate(invalid="ignore", over="ignore"):
                delta = a["_chill_portion_one_season"]((hr + 273.15).T)
            key = f"{cal}_{int(infill)}"
            out[f"daylen_{key}"] = dl
            keep = (np.arange(24 * n) // 24) % KEEP_EVERY == 0
            out[f"hourly_{key}"] = hr[keep]
            out[f"cp_{key}"] = np.sum(delta, axis=-1)
            out[f"cp_hours_{key}"] = np.sum(delta != 0, axis=-1)
    path = os.path.join(HERE, "ref_chill.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
