"""CUDA implementations behind ``xclim.core.calendar.percentile_doy`` / ``resample_doy``."""
from __future__ import annotations

import weakref

import numpy as np

from . import device
from .field import Field, attrs_of, dims_of, is_xarray, raw_values, time_axis_of, wrap_like
from .generic import _unwrap

# device-resident tables of the percentile arrays handed back to the caller, so that
# tx90p(tasmax, per) does not re-upload what percentile_doy just computed
_TABLE_CACHE: dict = {}


def _fingerprint(arr):
    """A few sampled values of a host array: detects in-place edits of a percentile array after
    ``percentile_doy`` handed it out (e.g. ``per.values -= 273.15``) at negligible cost."""
    if not isinstance(arr, np.ndarray) or arr.size == 0:
        return None
    flat = arr.reshape(-1) if arr.flags.c_contiguous else arr.ravel()[:0]
    if flat.size == 0:
        return None
    idx = np.linspace(0, flat.size - 1, 16).astype(np.int64)
    return flat[idx].tobytes()


def _remember_table(host_array, table_dev, meta=None):
    """Cache the doy-major device table of a percentile array handed to the caller, keyed by the
    identity of its values; ``meta`` = (other_dims, cell_shape) of the data the table was built from."""
    key = id(host_array)
    try:
        ref = weakref.ref(host_array, lambda _r, k=key: _TABLE_CACHE.pop(k, None))
    except TypeError:
        return
    _TABLE_CACHE[key] = (ref, table_dev, meta, _fingerprint(host_array))


def _recall_table(host_array, meta=None):
    hit = _TABLE_CACHE.get(id(host_array))
    if hit is None or hit[0]() is not host_array:
        return None
    if meta is not None and hit[2] is not None and tuple(hit[2]) != tuple(meta):
        return None                       # same values, other grid / dim order: rebuild from the values
    if hit[3] is not None and hit[3] != _fingerprint(host_array):
        _TABLE_CACHE.pop(id(host_array), None)   # edited in place since percentile_doy returned it
        return None
    return hit[1]


def year_ordinals(ta):
    years = np.unique(ta.year)
    return np.searchsorted(years, ta.year).astype(np.int16), years


def percentile_doy(arr, window=5, per=10.0, alpha=1.0 / 3.0, beta=1.0 / 3.0, copy=True):
    """Percentile value for each day of the year -- core/calendar.py:395-494.

    Returns dims ``(*space, dayofyear, percentiles)`` float64 with attrs ``climatology_bounds``,
    ``window``, ``alpha``, ``beta`` and a ``history`` entry naming ``percentile_doy`` (the
    bootstrap recognises the percentile argument by it, core/bootstrapping.py:131-135).  ``copy`` is
    accepted for signature parity; the input is never mutated.
    """
    x2d, cell_shape, other, ta = _unwrap(arr)
    pers = [float(per)] if np.isscalar(per) else [float(p) for p in per]
    yidx, years = year_ordinals(ta)
    n_doy = int(ta.doy.max())
    table = device.percentile_doy(x2d, ta.doy, yidx, n_doy, len(years), window, pers, alpha, beta)
    if n_doy == 366:  # core/calendar.py:484-485: drop doy 366, re-interpolate 1..365 onto 1..366
        table = _interp_each(table, len(pers))
    attrs = attrs_of(arr)
    attrs["climatology_bounds"] = [ta.date_strings(0)[0], ta.date_strings(len(ta) - 1)[0]]
    attrs["window"] = window
    attrs["alpha"] = alpha
    attrs["beta"] = beta
    hist = attrs.get("history", "")
    attrs["history"] = (hist + "\n" if hist else "") + (
        f"percentile_doy(arr, window={window}, per={pers}, alpha={alpha}, beta={beta}) - xclim_b200")
    nd = table.shape[1]
    # reference dim order: (*space, dayofyear, percentiles); transposed in HBM, not on the host
    vals = device.table_cell_major(table.contiguous()).reshape(cell_shape + (nd, len(pers)))
    from .options import OPTIONS
    host_t = vals if (OPTIONS["device_outputs"] and not is_xarray(arr)) else vals.cpu().numpy()
    out = wrap_like(arr, host_t, other + ("dayofyear", "percentiles"),
                    coords_extra={"dayofyear": np.arange(1, nd + 1), "percentiles": np.asarray(pers)},
                    attrs=attrs, name="per")
    _remember_table(out.values if isinstance(out, Field) else out.data, table, (tuple(other), tuple(cell_shape)))
    return out


def _stream_percentile_doy():
    global percentile_doy
    from .streaming import streamed
    percentile_doy = streamed(percentile_doy)


_stream_percentile_doy()


def _interp_each(table, n_per):
    import torch
    return torch.stack([device.doy_interp(table[i, :365].contiguous(), 1, 366) for i in range(n_per)])


def select_percentile(per_da, percentile=None):
    """``per.sel(percentiles=p)`` for Fields (xarray users call ``.sel`` themselves)."""
    if is_xarray(per_da):
        return per_da.sel(percentiles=percentile) if percentile is not None else per_da.squeeze("percentiles")
    dims = dims_of(per_da)
    ax = dims.index("percentiles")
    pcs = np.asarray(per_da.coords["percentiles"])
    i = 0 if percentile is None else int(np.nonzero(pcs == percentile)[0][0])
    vals = per_da.values[(slice(None),) * ax + (i,)]     # a view (numpy or device tensor): no copy of the table
    out = Field(vals, tuple(d for d in dims if d != "percentiles"), None,
                {k: v for k, v in per_da.coords.items() if k != "percentiles"}, dict(per_da.attrs), per_da.name)
    out.coords["percentiles"] = pcs[i]
    hit = _TABLE_CACHE.get(id(per_da.values))
    parent = _recall_table(per_da.values)
    if parent is not None:
        _remember_table(vals, parent[i:i + 1], hit[2])
    return out


def table_on_device(per_da, cell_shape, other_dims, dev):
    """(n_doy, C) float64 device table from a percentile array (dims ``(*space, dayofyear)``)."""
    import torch
    vals = raw_values(per_da)
    cached = _recall_table(vals, (tuple(other_dims), tuple(cell_shape)))
    if cached is not None and cached.shape[0] == 1 and cached.device == torch.device(dev):
        return cached[0]
    dims = dims_of(per_da)
    if "percentiles" in dims:
        ax = dims.index("percentiles")
        if vals.shape[ax] != 1:
            raise ValueError("select one percentile first: per.sel(percentiles=p)")
        vals = vals[(slice(None),) * ax + (0,)]
        dims = tuple(d for d in dims if d != "percentiles")
    if "dayofyear" not in dims:
        raise AttributeError("Source should have `dayofyear` coordinates.")  # core/calendar.py:781-782
    if hasattr(vals, "is_cuda"):       # a device-resident table in the reference's dim order
        space = tuple(d for d in dims if d != "dayofyear")
        t = vals.to(dev, torch.float64).movedim(dims.index("dayofyear"), 0)
        if space != tuple(other_dims):
            t = t.permute((0,) + tuple(1 + space.index(d) for d in other_dims))
        if tuple(t.shape[1:]) != tuple(cell_shape):
            raise ValueError(f"percentile array shape {tuple(t.shape[1:])} does not match the data grid {cell_shape}")
        return t.reshape(t.shape[0], -1).contiguous()
    space = tuple(d for d in dims if d != "dayofyear")
    h = np.asarray(vals, dtype=np.float64)
    if dims[-1] == "dayofyear" and space == tuple(other_dims) and h.flags.c_contiguous:
        # the reference layout (*space, dayofyear): upload as it lies and transpose in HBM (a host-side
        # transpose of the 3 GB full-grid table costs seconds)
        if tuple(h.shape[:-1]) != tuple(cell_shape):
            raise ValueError(f"percentile array shape {h.shape[:-1]} does not match the data grid {cell_shape}")
        n_doy = h.shape[-1]
        t = torch.from_numpy(h.reshape(-1, n_doy)).to(dev)           # (C, n_doy)
        return device.transpose_f64(t)                                # (n_doy, C)
    a = np.moveaxis(h, dims.index("dayofyear"), 0)
    if space != tuple(other_dims):
        a = np.transpose(a, (0,) + tuple(1 + space.index(d) for d in other_dims))
    if tuple(a.shape[1:]) != tuple(cell_shape):
        raise ValueError(f"percentile array shape {a.shape[1:]} does not match the data grid {cell_shape}")
    return torch.from_numpy(np.ascontiguousarray(a).reshape(a.shape[0], -1)).to(dev)


def adjust_table(table2d, ta):
    """core/calendar.py:729-760 (`adjust_doy_calendar`) on the device table; returns the table and
    the day-of-year index (1-based row + 1) of every time step."""
    max_t, min_t = int(ta.doy.max()), int(ta.doy.min())
    if table2d.shape[0] == ta.max_doy:
        return table2d, ta.doy
    tab = device.doy_interp(table2d, min_t, max_t)
    return tab, (ta.doy - min_t + 1)
