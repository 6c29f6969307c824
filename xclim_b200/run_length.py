"""CUDA implementations behind the signatures of ``xclim.indices.run_length``.

The reference functions take a boolean (or 0/1 float) mask ``da`` and a ``freq``; here the mask is
streamed once through the fused run-length kernel with the condition ``da > 0`` (``rle`` treats
every value > 0 as part of a run, indices/run_length.py:264-265).  For the fully fused
data-vs-threshold path use :func:`xclim_b200.generic.spell_length_statistics` /
:func:`xclim_b200.indices.maximum_consecutive_dry_days`, which never materialise the mask.
"""
from __future__ import annotations

import numpy as np

from . import _lib, device
from .field import attrs_of
from .generic import _unwrap, _wrap_periods

_GT = _lib.OPS[">"]


def _check(freq, index, ufunc_1dim):
    if ufunc_1dim is True and freq is not None:  # indices/run_length.py:67-68
        raise ValueError("Resampling after run length operations is not implemented for 1d method")
    if index not in ("first", "last"):
        raise ValueError(f"index must be 'first' or 'last', got {index!r}")


def _run_reduce(x2d, poff, reducer, window, resample_before_rl):
    """Run statistic of the mask ``x2d > 0``: named reducers, or "qNN" = quantile 0.NN of the run lengths
    (indices/run_length.py:320-327)."""
    if isinstance(reducer, str) and reducer.startswith("q") and reducer[1:].isdigit():
        return device.period_run_quantile(x2d, poff, _GT, 0.0, float(f"0.{reducer[1:]}"), window, resample_before_rl)
    if reducer not in _lib.RL_REDUCERS:
        raise NotImplementedError(f"reducer {reducer!r} is not supported by the xclim_b200 hot path")
    out, _ = device.period_runstat(x2d, poff, _GT, 0.0, _lib.RL_REDUCERS[reducer], window, resample_before_rl)
    return out


def _mask_unwrap(da):
    vals = da.values if not hasattr(da, "numpy") else da.values
    if getattr(vals, "dtype", None) is not None and str(vals.dtype) in ("bool", "torch.bool"):
        if hasattr(vals, "detach"):
            import torch
            da_vals = vals.to(torch.float32)
        else:
            da_vals = np.asarray(vals, dtype=np.float32)
        from .field import Field, is_xarray
        if is_xarray(da):
            da = da.astype(np.float32)
        else:
            da = Field(da_vals, da.dims, da.time, dict(da.coords), dict(da.attrs), da.name)
    return _unwrap(da)


def rle_statistics(da, reducer, window, dim="time", freq=None, ufunc_1dim="from_context", index="first"):
    """indices/run_length.py:275-335 with ``freq`` given (run-length THEN resample: each run is
    attributed with its full length to the period of its first element)."""
    if dim != "time":
        raise NotImplementedError("only dim='time' is supported")
    _check(freq, index, ufunc_1dim)
    x2d, cell_shape, other, ta = _mask_unwrap(da)
    poff = ta.period_offsets(freq)
    if index == "last" and freq is not None:
        # a run is attributed to the period of its LAST element (run_length.py:223-272): the same statistic on the
        # time-reversed series, whose runs start where the original ones end
        T = x2d.shape[0]
        out = _run_reduce(x2d.flip(0), (T - np.asarray(poff)[::-1]).astype(np.int32), reducer, window, False).flip(0)
    else:
        out = _run_reduce(x2d, poff, reducer, window, False)
    return _wrap_periods(da, out, cell_shape, other, ta, freq, attrs_of(da), dtype=np.float32)


def longest_run(da, dim="time", freq=None, ufunc_1dim="from_context", index="first"):
    """indices/run_length.py:338-378."""
    return rle_statistics(da, "max", 1, dim=dim, freq=freq, ufunc_1dim=ufunc_1dim, index=index)


def windowed_run_count(da, window, dim="time", freq=None, ufunc_1dim="from_context", index="first"):
    """indices/run_length.py:437-488: total length of runs at least ``window`` long."""
    return rle_statistics(da, "sum", window, dim=dim, freq=freq, ufunc_1dim=ufunc_1dim, index=index)


def windowed_run_events(da, window, dim="time", freq=None, ufunc_1dim="from_context", index="first"):
    """indices/run_length.py:381-434: number of runs at least ``window`` long."""
    return rle_statistics(da, "count", window, dim=dim, freq=freq, ufunc_1dim=ufunc_1dim, index=index)


def resample_and_rl(da, resample_before_rl, compute, *args, freq, dim="time", **kwargs):
    """indices/run_length.py:87-132.  ``compute`` must be one of this module's run statistics."""
    table = {rle_statistics: None, longest_run: ("max", 1), windowed_run_count: "sum", windowed_run_events: "count"}
    if compute not in table:
        raise NotImplementedError("resample_and_rl supports rle_statistics, longest_run, windowed_run_count/events")
    if compute is rle_statistics:
        reducer = kwargs.get("reducer", args[0] if args else None)
        window = kwargs.get("window", args[1] if len(args) > 1 else None)
    elif compute is longest_run:
        reducer, window = "max", 1
    else:
        reducer = table[compute]
        window = kwargs.get("window", args[0] if args else None)
    x2d, cell_shape, other, ta = _mask_unwrap(da)
    out = _run_reduce(x2d, ta.period_offsets(freq), reducer, window, bool(resample_before_rl))
    return _wrap_periods(da, out, cell_shape, other, ta, freq, attrs_of(da), dtype=np.float32)


def _boundary(da, window, dim, freq, coord, position):
    if dim != "time":
        raise NotImplementedError("only dim='time' is supported")
    if coord not in (False, None, "dayofyear"):
        raise NotImplementedError("coord must be False or 'dayofyear'")
    x2d, cell_shape, other, ta = _mask_unwrap(da)
    poff = ta.period_offsets(freq)
    out = device.period_boundary_run(x2d, poff, _GT, 0.0, window, last=(position == "last"))
    import torch
    vals = out.to(torch.float64)
    if coord == "dayofyear":  # lazy_indexing(time.dt.dayofyear, index), core/utils.py:202-276
        vals = index_to_doy(vals, poff, ta)
    return _wrap_periods(da, vals, cell_shape, other, ta, freq, attrs_of(da), dtype=np.float64)


def index_to_doy(vals, poff, ta):
    """(P, C) float64 device tensor of step indices relative to the period start (NaN = none) -> the
    day of year of that step, on the device (core/utils.py:202-276 ``lazy_indexing``)."""
    import torch
    dev = vals.device
    nan = torch.isnan(vals)
    start = torch.from_numpy(np.asarray(poff[:-1], dtype=np.int64)).to(dev)[:, None]
    idx = torch.where(nan, torch.zeros_like(vals), vals).to(torch.int64) + start
    doy = torch.from_numpy(np.asarray(ta.doy, dtype=np.float64)).to(dev)
    out = doy[idx.clamp_(0, len(ta) - 1)]
    return torch.where(nan, torch.full_like(out, float("nan")), out)


def first_run(da, window, dim="time", freq=None, coord=False, ufunc_1dim="from_context"):
    """indices/run_length.py:643-690: index of the first item of the first run of at least ``window``."""
    return _boundary(da, window, dim, freq, coord, "first")


def last_run(da, window, dim="time", freq=None, coord=False, ufunc_1dim="from_context"):
    """indices/run_length.py:693-740: index of the last item of the last run of at least ``window``."""
    return _boundary(da, window, dim, freq, coord, "last")


def windowed_max_run_sum(da, window, dim="time", freq=None, index="first"):
    """indices/run_length.py:491-540 for a non-negative float input (e.g. an excess over a threshold):
    largest run sum of the positive values over runs at least ``window`` long."""
    if dim != "time" or index != "first":
        raise NotImplementedError("only dim='time', index='first' are supported")
    x2d, cell_shape, other, ta = _mask_unwrap(da)
    out = device.period_run_maxsum(x2d, ta.period_offsets(freq), _GT, 0.0, window, resample_before_rl=False)
    return _wrap_periods(da, out, cell_shape, other, ta, freq, attrs_of(da), dtype=np.float32)
