"""Chill portions (Dynamic Model), chill units (Utah Model) and the hourly temperature they take.

The reference builds the hourly series of ``make_hourly_temperature`` (indices/helpers.py:1059-1123) as a float64
array 24 times the size of its daily inputs, and ``_chill_portion_one_season`` (indices/_agro.py:1436-1465) then
loops over every hour in Python.  Here ``make_hourly_temperature`` returns a lazy :class:`HourlyTemperature` that
records its daily inputs; the chill functions recognise it and run one fused kernel pass that makes each day's 24
hours in registers (``xc_chill_daily_f32``).  Explicit hourly series (24 steps per day from 00:00) go through the
same kernel reading the hours (``xc_chill_hourly``).  Anything that reads a lazy series' values materialises it
once, as float64, with ``xc_hourly_temperature_f32``.
"""
from __future__ import annotations

import numpy as np

from . import _lib, device
from .field import Field, dims_of, is_xarray, raw_values
from .generic import _unwrap, _wrap_periods
from .options import OPTIONS
from .timeaxis import TimeAxis
from .units import units_of


# ------------------------------------------------------------------------------------------ hourly time axis
class HourlyAxis:
    """An hourly time axis of 24 regular steps per day from 00:00: the daily :class:`TimeAxis` ``days`` plus the
    hour; the last day may be partial (``n_hours``)."""

    def __init__(self, days: TimeAxis, n_hours: int | None = None, coord=None):
        self.days = days
        self.n_hours = 24 * len(days) if n_hours is None else int(n_hours)
        if not 24 * (len(days) - 1) < self.n_hours <= 24 * len(days):
            raise ValueError(f"{self.n_hours} hours do not fall on {len(days)} days")
        self.coord = coord

    @classmethod
    def hourly(cls, start: str, n_hours: int, calendar: str = "standard") -> "HourlyAxis":
        """``n_hours`` consecutive hours from ``start`` ("YYYY-MM-DD") at 00:00."""
        return cls(TimeAxis.daily(start, -(-int(n_hours) // 24), calendar), n_hours)

    @classmethod
    def from_xarray(cls, time) -> "HourlyAxis":
        dt = time.dt
        hour, minute, second = (np.asarray(getattr(dt, k).values) for k in ("hour", "minute", "second"))
        n = hour.size
        if n == 0 or minute.any() or second.any() or not np.array_equal(hour, np.arange(n) % 24):
            raise NotImplementedError("hourly inputs must hold 24 regular steps per day starting at 00:00")
        days = TimeAxis.from_xarray(time[::24])
        _check_gap_free(days)
        return cls(days, n, coord=time)

    def __len__(self) -> int:
        return self.n_hours

    @property
    def calendar(self) -> str:
        return self.days.calendar


def _check_gap_free(days):
    from .converters import _check_daily
    try:
        _check_daily(days)
    except NotImplementedError:
        raise NotImplementedError("hourly inputs must hold 24 regular steps per day, without gaps") from None


def _hourly_axis(tas):
    if isinstance(tas, HourlyTemperature):
        return tas.time
    if is_xarray(tas):
        return HourlyAxis.from_xarray(tas["time"])
    if isinstance(tas, Field) and isinstance(tas.time, HourlyAxis):
        return tas.time
    raise NotImplementedError("chill_portions and chill_units take hourly temperature: an HourlyAxis-labelled "
                              "Field, an hourly DataArray or the result of make_hourly_temperature")


# ------------------------------------------------------------------------------------------ lazy hourly series
class HourlyTemperature(Field):
    """The hourly temperature of ``make_hourly_temperature``, kept as its daily inputs: ``tasmin`` and ``tasmax``
    (Fields of the same dims), ``lat`` (per-cell latitudes in degrees north, labelled by the spatial dims) and
    ``infill_polar_days``.  ``values`` materialises the (24 T, ...) float64 series once."""

    def __init__(self, tasmin, tasmax, lat, infill_polar_days):
        self.tasmin, self.tasmax, self.lat = tasmin, tasmax, lat
        self.infill_polar_days = bool(infill_polar_days)
        self.dims = tuple(tasmin.dims)
        self.time = HourlyAxis(tasmin.time)
        self.coords = {k: v for k, v in tasmin.coords.items() if k != "time"}
        self.attrs = {"units": units_of(tasmin)}
        self.name = None
        self._values = None

    @property
    def values(self):
        if self._values is None:
            self._values = _materialise(self.tasmin, self.tasmax, self.lat, self.infill_polar_days)
        return self._values

    @property
    def shape(self):
        s = list(self.tasmin.shape)
        s[self.dims.index("time")] *= 24
        return tuple(s)

    @property
    def dtype(self):
        return np.dtype(np.float64)


def _weights(ta, lat, other, cell_shape, infill, dev):
    """Device weight rows (T, L, CHILL_ROW) of the distinct latitudes and the (C,) row index of every cell."""
    import torch

    from .converters import hourly_weights
    from .fire import _per_cell
    lat_c = _per_cell(lat, other, cell_shape, np.float64, "lat")
    lat_u, idx = np.unique(lat_c, return_inverse=True)
    w = torch.from_numpy(hourly_weights(ta, lat_u, infill)).to(dev)
    return w, torch.from_numpy(idx.astype(np.int32).reshape(-1)).to(dev)


def _materialise(tasmin, tasmax, lat, infill):
    import torch
    lo, cell_shape, other, ta = _unwrap(tasmin)
    hi, _, _, _ = _unwrap(tasmax)
    w, idx = _weights(ta, lat, other, cell_shape, infill, lo.device)
    out = device.hourly_temperature(lo, hi, w, idx).reshape((24 * len(ta),) + cell_shape)
    tpos = dims_of(tasmin).index("time")
    out = torch.movedim(out, 0, tpos)
    on_device = hasattr(raw_values(tasmin), "is_cuda") and raw_values(tasmin).is_cuda
    return out if on_device else out.cpu().numpy()


def _broadcast_fields(a, b):
    """Two Fields over the union of their dims (the larger one's order), as ``xr.merge`` and arithmetic do."""
    if tuple(a.dims) == tuple(b.dims):
        return a, b
    a_big = len(a.dims) >= len(b.dims)
    big, small = (a, b) if a_big else (b, a)
    if not set(small.dims) <= set(big.dims):
        raise ValueError(f"tasmin and tasmax dims {tuple(a.dims)} and {tuple(b.dims)} cannot be broadcast")
    v = np.asarray(raw_values(small))
    order = sorted(range(len(small.dims)), key=lambda i: big.dims.index(small.dims[i]))
    v = np.transpose(v, order)
    shape = [1] * len(big.dims)
    for d, n in zip([small.dims[i] for i in order], v.shape):
        shape[big.dims.index(d)] = n
    v = np.ascontiguousarray(np.broadcast_to(v.reshape(shape), big.shape))
    coords = {**small.coords, **big.coords}
    grown = Field(v, tuple(big.dims), big.time, coords, dict(small.attrs), small.name)
    big = Field(big.values, tuple(big.dims), big.time, coords, dict(big.attrs), big.name)
    return (big, grown) if a_big else (grown, big)


def make_hourly_temperature(tasmin, tasmax, infill_polar_days=False):
    """Hourly temperature from daily ``tasmin`` and ``tasmax`` -- indices/helpers.py:1059-1123 (Linvill 1990).

    A sine from tasmin at sunrise (00:00) to tasmax two hours before sunset, then a logarithmic decrease toward
    the next day's tasmin (the last day's own).  The day length comes from the ``lat`` coordinate
    (``day_lengths``); polar days and nights are NaN, or 24 h and 0 h with ``infill_polar_days``.  Inputs named
    ``tasmin`` / ``tasmax`` are taken by name, as the reference's ``xr.merge`` does, whatever their order.  Field
    inputs give a lazy :class:`HourlyTemperature` that the chill functions run from the daily values; DataArray
    inputs give the materialised float64 DataArray.  Both inputs must carry the same units."""
    if getattr(tasmin, "name", None) == "tasmax" and getattr(tasmax, "name", None) == "tasmin":
        tasmin, tasmax = tasmax, tasmin
    if units_of(tasmin) != units_of(tasmax):
        raise ValueError(f"tasmin and tasmax must share their units, got {units_of(tasmin)!r} and "
                         f"{units_of(tasmax)!r}")
    from .converters import _gather_lat
    from .fire import _label_per_cell
    if is_xarray(tasmin) or is_xarray(tasmax):
        import xarray as xr
        tasmin, tasmax = xr.broadcast(tasmin, tasmax)
        lat = tasmin.coords["lat"] if "lat" in tasmin.coords else _gather_lat(tasmax, "make_hourly_temperature")
        lo = Field(np.asarray(tasmin.values), tuple(tasmin.dims), HourlyAxis(_daily_axis(tasmin)).days, {}, {})
        hi = Field(np.asarray(tasmax.transpose(*tasmin.dims).values), lo.dims, lo.time, {}, {})
        vals = _materialise(lo, hi, _lat_field(lat, tasmin), infill_polar_days)
        days = lo.time
        n = 24 * len(days)
        time = xr.date_range(f"{days.date_strings(0)[0]}", periods=n, freq="h", calendar=days.calendar,
                             use_cftime=days.calendar not in ("standard", "gregorian", "proleptic_gregorian"))
        coords = {d: tasmin.coords[d] for d in tasmin.dims if d != "time" and d in tasmin.coords}
        coords["time"] = time
        return xr.DataArray(vals, dims=tasmin.dims, coords=coords, attrs={"units": units_of(tasmin)})
    tasmin, tasmax = _broadcast_fields(tasmin, tasmax)
    if "lat" in tasmin.coords:
        lat = tasmin.coords["lat"]
        lat = Field(np.asarray(getattr(lat, "values", lat), np.float64), ("lat",), None, {}, {})
    else:
        lat = _gather_lat(tasmin, "make_hourly_temperature")
    if "lat" not in tasmin.dims and np.asarray(raw_values(lat)).size == 1:
        lat = float(np.asarray(raw_values(lat)).reshape(-1)[0])     # a scalar latitude for every cell
    return HourlyTemperature(tasmin, tasmax, _label_per_cell(lat, tasmin), infill_polar_days)


def _daily_axis(da):
    return TimeAxis.from_xarray(da["time"])


def _lat_field(lat, template):
    return Field(np.asarray(lat.values, np.float64), tuple(lat.dims), None, {}, {})


# ------------------------------------------------------------------------------------------ kernels per call
def _run(x, tasmax, lat, *, poff, mask, to_k, to_c, what, infill, days, freq, name, attrs):
    """One kernel pass: the fused one when ``tasmax`` is given (``x`` is then tasmin), else over the hourly ``x``.
    Returns ``(result, valid)`` labelled per period (``valid``: selected non-NaN hours, float64)."""
    if tasmax is not None:
        lo, cell_shape, other, ta = _unwrap(x)
        hi, _, _, _ = _unwrap(tasmax)
        w, idx = _weights(ta, lat, other, cell_shape, infill, lo.device)
        cp, cu, valid = device.chill_daily(lo, hi, w, idx, poff, mask, to_k, to_c, what, want_valid=True)
    else:
        x2d, cell_shape, other = _unwrap_hourly(x)
        cp, cu, valid = device.chill_hourly(x2d, poff, mask, to_k, to_c, what, want_valid=True)
    out = cp if what & _lib.CHILL_PORTIONS else cu
    return (_wrap_periods(x, out, cell_shape, other, days, freq, dict(attrs), dtype=np.float64, name=name),
            _wrap_periods(x, valid, cell_shape, other, days, freq, {}, dtype=np.float64, name="valid"))


def _unwrap_hourly(da):
    """(H, C) device tensor of an hourly input, float64 kept as float64, anything else as float32."""
    dims = dims_of(da)
    tpos = dims.index("time")
    v = raw_values(da)
    if str(v.dtype) in ("float64", "torch.float64"):
        x2d, cell_shape = device.to_time_cell_f64(v, tpos)
    else:
        x2d, cell_shape = device.to_time_cell(v, tpos)
    return x2d, cell_shape, tuple(d for d in dims if d != "time")


def _affine(tas, target):
    from .fire import _affine as affine
    return affine(tas, target)


def _chill(tas, freq, what, indexer, drop):
    """``(result, valid, expected_hours, kept_periods)`` of one chill call (see :func:`chill_portions`)."""
    from .streaming import streamed
    hax = _hourly_axis(tas)
    days = hax.days
    poff = days.period_offsets(freq)
    mask = days.select_mask(**indexer) if indexer else None
    kw = dict(poff=poff, mask=mask, to_k=_affine(tas, "K"), to_c=_affine(tas, "degC"), what=what, days=days,
              freq=freq, name="cp" if what & _lib.CHILL_PORTIONS else "cu", attrs={"units": ""})
    if isinstance(tas, HourlyTemperature):
        out, valid = streamed(_run)(tas.tasmin, tas.tasmax, tas.lat, infill=tas.infill_polar_days, **kw)
    else:
        if len(hax) != _time_len(tas):
            raise ValueError("the hourly axis does not match the input's time dimension")
        out, valid = streamed(_run)(tas, None, None, infill=False, **kw)
    expected = days.expected_period_lengths(freq, **indexer) * 24
    keep = slice(0, len(poff) - 1)
    if drop and mask is not None:      # select_time(drop=True): the periods run from the first selected day's
        n_sel = np.add.reduceat(mask.astype(np.int64), poff[:-1])
        hit = np.nonzero(n_sel)[0]
        if hit.size == 0:
            raise ValueError("the indexer selects no day of the series")
        keep = slice(int(hit[0]), int(hit[-1]) + 1)
        empty = n_sel[keep] == 0         # a period between them without a selected day is NaN
        out = _set_periods(_isel_periods(out, keep), empty)
        valid = _isel_periods(valid, keep)
        expected = expected[keep]
    return out, valid, expected


def _time_len(da):
    return int(da.shape[dims_of(da).index("time")])


def _isel_periods(f, sl):
    if is_xarray(f):
        return f.isel(time=sl)
    idx = [slice(None)] * len(f.dims)
    idx[f.dims.index("time")] = sl
    coords = dict(f.coords)
    if "time" in coords:
        coords["time"] = np.asarray(coords["time"])[sl]
    return Field(f.values[tuple(idx)], f.dims, None, coords, dict(f.attrs), f.name)


def _set_periods(f, empty):
    if not empty.any():
        return f
    v = raw_values(f)
    shape = [1] * len(f.dims)
    shape[f.dims.index("time")] = empty.size
    m = empty.reshape(shape)
    if hasattr(v, "is_cuda"):
        import torch
        v = torch.where(torch.from_numpy(m).to(v.device), torch.full_like(v, float("nan")), v)
    else:
        v = np.where(m, np.nan, v)
    return f.copy(data=v) if is_xarray(f) else Field(v, f.dims, f.time, dict(f.coords), dict(f.attrs), f.name)


def chill_portions(tas, freq="YS", **indexer):
    """Chill portions after the Dynamic Model -- indices/_agro.py:1494-1534 (Fishman et al. 1987, Luedeling et al.
    2009), float64 per period of ``freq``, on hourly ``tas``.  ``indexer`` is ``select_time(drop=True)``: the
    recurrence runs over the selected hours only, without restarting at a gap, and the periods run from the first
    to the last one holding a selected day.  One kernel pass; the sums follow DESIGN.md section 4."""
    return _chill(tas, freq, _lib.CHILL_PORTIONS, indexer, drop=True)[0]


def chill_units(tas, positive_only=False, freq="YS"):
    """Chill units after the Utah Model -- indices/_agro.py:1537-1592 (Richardson et al. 1974), float64 per period
    of ``freq``, on hourly ``tas``; NaN hours are left out, and with ``positive_only`` only days whose sum is
    positive count."""
    what = _lib.CHILL_UNITS | (_lib.CHILL_POSITIVE_ONLY if positive_only else 0)
    return _chill(tas, freq, what, {}, drop=False)[0]


# ------------------------------------------------------------------------------------------ indicators
def _yearly(freq):
    from .timeaxis import parse_offset
    if parse_offset(freq)[1] != "Y":
        raise ValueError(f"Resampling frequency {freq} is not allowed for this indicator. The following are "
                         "allowed: ['Y'].")


def _indicator(res, name):
    out, valid, expected = res
    method = OPTIONS["check_missing"]
    if method not in ("any", "skip"):
        raise NotImplementedError(f"check_missing={method!r} is not supported for hourly indicators")
    v = raw_values(out)
    shape = [1] * len(out.dims)
    shape[out.dims.index("time")] = expected.size
    exp = expected.reshape(shape).astype(np.float64)
    if method == "any":
        val = raw_values(valid)
        if hasattr(v, "is_cuda"):
            import torch
            v = torch.where(val != torch.from_numpy(exp).to(v.device), torch.full_like(v, float("nan")), v)
        else:
            v = np.where(np.asarray(val) != exp, np.nan, v)
    attrs = {**dict(out.attrs), "units": "1"}
    if is_xarray(out):
        return out.copy(data=v).assign_attrs(attrs).rename(name)
    return Field(v, out.dims, out.time, dict(out.coords), attrs, name)


def atmos_chill_portions(tas, freq="YS", **indexer):
    """``xclim.atmos.chill_portions`` (identifier ``cp``, indicators/atmos/_temperature.py:1577-1597): yearly
    periods only, NaN where a period misses a selected hour (MissingAny on the hourly steps)."""
    _yearly(freq)
    return _indicator(_chill(tas, freq, _lib.CHILL_PORTIONS, indexer, drop=True), "cp")


def atmos_chill_units(tas, positive_only=False, freq="YS", **indexer):
    """``xclim.atmos.chill_units`` (identifier ``cu``, :1599-1610): the indicator's indexer makes the unselected
    hours NaN; yearly periods only, NaN where a period misses a selected hour."""
    _yearly(freq)
    what = _lib.CHILL_UNITS | (_lib.CHILL_POSITIVE_ONLY if positive_only else 0)
    return _indicator(_chill(tas, freq, what, indexer, drop=False), "cu")


__all__ = ["HourlyAxis", "HourlyTemperature", "make_hourly_temperature", "chill_portions", "chill_units"]
