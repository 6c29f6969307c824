"""CUDA implementation behind ``xclim.indices.fire`` (Canadian Forest Fire Weather Index System).

SURVEY.md section 8(f).4.  The reference runs ``_fire_weather_calc`` (indices/fire/_cffwis.py:680-873) -- a
Python loop over days around numba ufuncs -- per dask chunk through ``xr.apply_ufunc``
(``fire_weather_ufunc``, :879-1151).  Here the whole day loop, the season masks, overwintering and the dry
starts are ONE kernel (``xc_fwi_f32``): a lane walks a grid cell through time and writes every requested
output in the same pass.  The functions keep the reference's names, argument meaning and errors:

* :func:`fire_weather_ufunc` (:879-1151) -- no unit handling, inputs in degC, mm/day, %, km/h, m;
* :func:`cffwis_indices` (:1273-1402), :func:`drought_code` (:1415-1500), :func:`duff_moisture_code`
  (:1513-1594) -- unit-aware: the conversion of the input arrays is folded into the kernel's loads;
* :func:`fire_season` (:1609-1691, ``freq=None``);
* the element-wise members :func:`initial_spread_index`, :func:`build_up_index`, :func:`fire_weather_index`,
  :func:`daily_severity_rating` (:449-546) and :func:`overwintering_drought_code` (:1165-1250).
"""
from __future__ import annotations

from collections import namedtuple

import numpy as np

from . import device
from .field import Field, dims_of, is_xarray, raw_values, wrap_like
from .generic import _unwrap
from .options import OPTIONS
from .units import convert_units_to, units_of

#: ``default_params`` of the reference (:161-178): value, or (value, units)
default_params = {
    "temp_start_thresh": (12.0, "degC"),
    "temp_end_thresh": (5.0, "degC"),
    "snow_thresh": (0.01, "m"),
    "temp_condition_days": 3,
    "snow_condition_days": 3,
    "carry_over_fraction": 0.75,
    "wetting_efficiency_fraction": 0.75,
    "dc_start": 15,
    "dmc_start": 6,
    "ffmc_start": 85,
    "prec_thresh": (1.0, "mm/d"),
    "dc_dry_factor": 5,
    "dmc_dry_factor": 2,
    "snow_cover_days": 60,
    "snow_min_cover_frac": 0.75,
    "snow_min_mean_depth": (0.1, "m"),
}

_ORDER = ["DC", "DMC", "FFMC", "ISI", "BUI", "FWI", "DSR"]
_LENGTH = {"m": 1.0, "cm": 0.01, "mm": 0.001, "km": 1000.0}
_IDENTITY = (1.0, 0.0)


def _affine(da, target):
    """``(scale, offset)`` with ``value[target] = raw * scale + offset`` for the units of ``da``."""
    u = units_of(da).strip()
    if target == "m":
        if u not in _LENGTH:
            raise ValueError(f"Cannot convert {u!r} to 'm'")
        return (_LENGTH[u], 0.0)
    if target == "%":
        if u in ("%", "percent"):
            return _IDENTITY
        if u in ("", "1"):
            return (100.0, 0.0)
        raise ValueError(f"Cannot convert {u!r} to '%'")
    zero = convert_units_to(f"0 {u}", target)
    one = convert_units_to(f"1 {u}", target)
    return (one - zero, zero)


def _param_value(name, value):
    """Keyword parameter in the units ``default_params`` names (``_convert_parameters``, :1252-1263)."""
    default = default_params[name]
    if isinstance(default, tuple):
        if isinstance(value, str):
            return _length_or(value, default[1])
        return float(value)
    return value


def _length_or(q, target):
    if target == "m":
        from .units import parse_quantity
        val, u = parse_quantity(q)
        if u is None:
            return val
        if u not in _LENGTH:
            raise ValueError(f"Cannot convert {u!r} to 'm'")
        return val * _LENGTH[u]
    return convert_units_to(q, target)


def _convert_parameters(params, funcname="fire weather indices"):
    out = {}
    for k, v in params.items():
        if k not in default_params:
            raise ValueError(f"{k} is not a valid parameter for {funcname}. See the docstring of the function "
                             "and the list in xc.indices.fire.default_params.")
        out[k] = _param_value(k, v)
    return out


def _per_cell(obj, template_dims, cell_shape, dtype, name):
    """A per-cell input (previous codes, latitude) broadcast to the flattened cell axis, as a host array."""
    if obj is None:
        return None
    if isinstance(obj, Field) or is_xarray(obj):
        vals = raw_values(obj)
        if hasattr(vals, "detach"):
            vals = vals.detach().cpu().numpy()
        vals = np.asarray(vals)
        dims = dims_of(obj)
        if "time" in dims:
            raise ValueError(f"`{name}` must not have a time dimension")
        shape = [1] * len(template_dims)
        for d, n in zip(dims, vals.shape):
            if d not in template_dims:
                raise ValueError(f"`{name}` has a dimension `{d}` that the series do not have")
            shape[template_dims.index(d)] = n
        order = sorted(range(len(dims)), key=lambda i: template_dims.index(dims[i]))
        vals = np.transpose(vals, order).reshape(shape)
    else:
        vals = np.asarray(obj)
    return np.array(np.broadcast_to(vals, cell_shape), dtype=dtype).reshape(-1)


def _to_device(host, dev):
    import torch
    return None if host is None else torch.from_numpy(host).to(dev)


def _run(series, affine, lat, state, season_mask, outputs, season_method, overwintering, dry_start,
         initial_start_up, params):
    """Unwrap, call the kernel, wrap.  ``series``: dict tas/pr/hurs/ws/snd -> labelled array or None."""
    template = series["tas"] if series["tas"] is not None else series["pr"]
    x = {}
    cell_shape = other = ta = None
    for k, da in series.items():
        if da is None:
            x[k] = None
            continue
        x2d, cs, od, t = _unwrap(da)
        if cell_shape is None:
            cell_shape, other, ta = cs, od, t
        elif cs != cell_shape or x2d.shape != next(v for v in x.values() if v is not None).shape:
            raise ValueError("the input series must share their shape")
        x[k] = x2d
    dev = next(v for v in x.values() if v is not None).device
    lat_h = _per_cell(lat, other, cell_shape, np.float64, "lat")
    if lat_h is not None and np.any((lat_h > 90) | (lat_h < -90)):
        raise ValueError("Invalid lat specified.")
    st = {k: _to_device(_per_cell(v, other, cell_shape, np.float32, k), dev) for k, v in state.items()}
    mask_d = None
    if season_mask is not None:
        m2d, cs, _, _ = _unwrap_mask(season_mask)
        if cs != cell_shape:
            raise ValueError("season_mask must share the shape of the series")
        mask_d = m2d.to(dev)
    P = device.fwi_params(season_method, overwintering, dry_start, initial_start_up, in_affine=affine, **params)
    month = np.asarray(ta.month, dtype=np.int8)
    res = device.fire_weather(x["tas"], x["pr"], x["hurs"], x["ws"], x["snd"], month, lat_h, mask_d, st["dc0"],
                              st["dmc0"], st["ffmc0"], st["winter_pr"], outputs, P)
    out = {}
    keep_dev = OPTIONS["device_outputs"] and not is_xarray(template)
    time = ta if ta.coord is None else ta.coord
    for name, t in res.items():
        if name == "winter_pr":
            vals = t.reshape(cell_shape)
            vals = vals if keep_dev else vals.cpu().numpy()
            out[name] = wrap_like(template, vals, tuple(other), attrs={}, name=name)
            continue
        vals = t.contiguous().reshape((t.shape[0],) + cell_shape)
        if name == "season_mask":
            vals = vals.bool()
        vals = vals if keep_dev else vals.cpu().numpy()
        out[name] = wrap_like(template, vals, ("time",) + tuple(other), time=time, attrs={}, name=name)
    return out


def _unwrap_mask(mask):
    """(T, C) uint8 tensor of a boolean season mask."""
    import torch
    dims = dims_of(mask)
    if "time" not in dims:
        raise ValueError("season_mask must have a `time` dimension")
    v = raw_values(mask)
    if hasattr(v, "detach"):
        t = v.movedim(dims.index("time"), 0).to(torch.uint8)
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.moveaxis(np.asarray(v), dims.index("time"), 0)).astype(np.uint8))
    cell_shape = tuple(t.shape[1:])
    return t.reshape(t.shape[0], -1).contiguous(), cell_shape, None, None


def _label_per_cell(obj, template):
    """Per-cell arguments given as bare arrays get the spatial dims of the series, so that the slab streamer
    can cut them along the leading spatial dimension together with the series."""
    if obj is None or isinstance(obj, Field) or is_xarray(obj):
        return obj
    space = tuple(d for d in dims_of(template) if d != "time")
    shape = tuple(n for d, n in zip(dims_of(template), template.shape) if d != "time")
    a = np.asarray(obj)
    if a.shape == shape:
        return Field(a, space, None, {}, {})
    if a.ndim == 1 and space and a.shape[0] == shape[0]:
        return Field(a, space[:1], None, {}, {})
    return obj                                   # scalars and other broadcastable shapes: used whole


def fire_weather_ufunc(*, tas, pr, hurs=None, sfcWind=None, snd=None, lat=None, dc0=None, dmc0=None, ffmc0=None,
                       winter_pr=None, season_mask=None, start_dates=None, indexes=None, season_method=None,
                       overwintering=False, dry_start=None, initial_start_up=True, _affine_of=None, **params):
    """Fire weather indexes, no unit handling -- indices/fire/_cffwis.py:879-1151.

    ``tas`` degC, ``pr`` mm/day, ``hurs`` %, ``sfcWind`` km/h, ``snd`` m.  Returns a dict of the indexes
    asked for plus the ones they depend on (:1046-1057), ``season_mask`` when it is computed here and
    ``winter_pr`` under overwintering, like the reference.  Host-backed series beyond the streaming
    threshold go through the slab streamer (every output is assembled on the host slab by slab), as for
    the other indices.
    """
    from .streaming import streamed
    lat, dc0, dmc0, ffmc0, winter_pr = (_label_per_cell(v, tas) for v in (lat, dc0, dmc0, ffmc0, winter_pr))
    return streamed(_fire_weather)(tas=tas, pr=pr, hurs=hurs, sfcWind=sfcWind, snd=snd, lat=lat, dc0=dc0, dmc0=dmc0,
                                   ffmc0=ffmc0, winter_pr=winter_pr, season_mask=season_mask, indexes=indexes,
                                   season_method=season_method, overwintering=overwintering, dry_start=dry_start,
                                   initial_start_up=initial_start_up, _affine_of=_affine_of, **params)


def _fire_weather(*, tas, pr, hurs=None, sfcWind=None, snd=None, lat=None, dc0=None, dmc0=None, ffmc0=None,
                  winter_pr=None, season_mask=None, indexes=None, season_method=None, overwintering=False,
                  dry_start=None, initial_start_up=True, _affine_of=None, **params):
    want = set(indexes or _ORDER)
    unknown = want - set(_ORDER)
    if unknown:
        raise ValueError(f"unknown indexes {sorted(unknown)}")
    for idx, needs in (("DSR", {"FWI"}), ("FWI", {"ISI", "BUI"}), ("BUI", {"DC", "DMC"}), ("ISI", {"FFMC"})):
        if idx in want:
            want |= needs
    outputs = sorted(want, key=_ORDER.index)
    # which inputs the indexes and the season method need (:1059-1081)
    needed = (
        (tas, "tas", ["DC", "DMC", "FFMC", "WF93", "LA08"]),
        (pr, "pr", ["DC", "DMC", "FFMC"]),
        (hurs, "hurs", ["DMC", "FFMC"]),
        (sfcWind, "sfcWind", ["FFMC"]),
        (snd, "snd", ["LA08"]),
        (lat, "lat", ["DC", "DMC"]),
    )
    used = {}
    for arg, name, usedby in needed:
        if any(ind in outputs + [season_method] for ind in usedby):
            if arg is None:
                raise TypeError(f"Missing input argument {name} for index combination {outputs} "
                                f"with fire season method '{season_method}'.")
            used[name] = arg
    if snd is not None and dry_start == "GFWED":
        used["snd"] = snd
        dry_start = "GFWED+SNOW"
    elif dry_start not in (None, "CFS", "GFWED"):
        raise ValueError("'dry_start' must be one of None, 'CFS' or 'GFWED'.")
    if season_method == "GFWED" and snd is not None:
        used["snd"] = snd                   # _fire_season reads it (:661-668) though the check above does not ask
    if season_mask is not None:
        season_method = "mask"
    elif season_method is not None:
        if season_method not in ("WF93", "LA08", "GFWED"):
            raise ValueError("`method` must be one of 'WF93', 'LA08' or 'GFWED'.")
        outputs.append("season_mask")
    if overwintering:
        if season_method is None:
            raise ValueError("If overwintering is activated, either `season_method` or `season_mask` must be given.")
        outputs.append("winter_pr")
    kw = {k: (v if not isinstance(v, tuple) else v[0]) for k, v in default_params.items()}
    unknown = set(params) - set(default_params)
    if unknown:
        raise TypeError(f"fire_weather_ufunc() got unexpected keyword arguments {sorted(unknown)}")
    kw.update(params)
    series = {"tas": used.get("tas", tas), "pr": used.get("pr"), "hurs": used.get("hurs"), "ws": used.get("sfcWind"),
              "snd": used.get("snd")}
    affine = _affine_of or [_IDENTITY] * 5
    state = {"dc0": dc0, "dmc0": dmc0, "ffmc0": ffmc0, "winter_pr": winter_pr if overwintering else None}
    return _run(series, affine, used.get("lat"), state, season_mask, outputs, season_method, overwintering, dry_start,
                initial_start_up, kw)


def _unitless(out):
    for f in out.values():
        f.attrs["units"] = ""
    return out


CFFWISIndices = namedtuple("CFFWISIndices", ["DC", "DMC", "FFMC", "ISI", "BUI", "FWI"])


def cffwis_indices(tas, pr, sfcWind, hurs, lat, snd=None, ffmc0=None, dmc0=None, dc0=None, season_mask=None,
                   season_method=None, overwintering=False, dry_start=None, initial_start_up=True, **params):
    """The six Canadian Fire Weather Index System indices -- indices/fire/_cffwis.py:1273-1402."""
    affine = [_affine(tas, "degC"), _affine(pr, "mm/d"), _affine(hurs, "%"), _affine(sfcWind, "km/h"),
              _affine(snd, "m") if snd is not None else _IDENTITY]
    out = fire_weather_ufunc(tas=tas, pr=pr, hurs=hurs, sfcWind=sfcWind, lat=lat, dc0=dc0, dmc0=dmc0, ffmc0=ffmc0,
                             snd=snd, indexes=["DC", "DMC", "FFMC", "ISI", "BUI", "FWI"], season_mask=season_mask,
                             season_method=season_method, overwintering=overwintering, dry_start=dry_start,
                             initial_start_up=initial_start_up, _affine_of=affine, **_convert_parameters(params))
    _unitless(out)
    return CFFWISIndices(*(out[k] for k in CFFWISIndices._fields))


def drought_code(tas, pr, lat, snd=None, dc0=None, season_mask=None, season_method=None, overwintering=False,
                 dry_start=None, initial_start_up=True, **params):
    """Drought code -- indices/fire/_cffwis.py:1415-1500."""
    affine = [_affine(tas, "degC"), _affine(pr, "mm/d"), _IDENTITY, _IDENTITY,
              _affine(snd, "m") if snd is not None else _IDENTITY]
    out = fire_weather_ufunc(tas=tas, pr=pr, lat=lat, dc0=dc0, snd=snd, indexes=["DC"], season_mask=season_mask,
                             season_method=season_method, overwintering=overwintering, dry_start=dry_start,
                             initial_start_up=initial_start_up, _affine_of=affine,
                             **_convert_parameters(params, "drought_code"))
    return _unitless(out)["DC"]


def duff_moisture_code(tas, pr, hurs, lat, snd=None, dmc0=None, season_mask=None, season_method=None, dry_start=None,
                       initial_start_up=True, **params):
    """Duff moisture code -- indices/fire/_cffwis.py:1513-1594."""
    affine = [_affine(tas, "degC"), _affine(pr, "mm/d"), _affine(hurs, "%"), _IDENTITY,
              _affine(snd, "m") if snd is not None else _IDENTITY]
    out = fire_weather_ufunc(tas=tas, pr=pr, hurs=hurs, lat=lat, dmc0=dmc0, snd=snd, indexes=["DMC"],
                             season_mask=season_mask, season_method=season_method, dry_start=dry_start,
                             initial_start_up=initial_start_up, _affine_of=affine,
                             **_convert_parameters(params, "duff_moisture_code"))
    return _unitless(out)["DMC"]


def fire_season(tas, snd=None, method="WF93", freq=None, temp_start_thresh="12 degC", temp_end_thresh="5 degC",
                temp_condition_days=3, snow_condition_days=3, snow_thresh="0.01 m"):
    """Fire season mask -- indices/fire/_cffwis.py:1609-1691 (every season, ``freq=None``)."""
    if freq is not None:
        raise NotImplementedError("fire_season(freq=...) (longest season per period) is not part of the xclim_b200 hot path")
    if not all(np.isscalar(v) for v in (temp_start_thresh, temp_end_thresh, snow_thresh)):
        raise ValueError("Thresholds must be scalar.")
    if method not in ("WF93", "LA08", "GFWED"):
        raise ValueError("`method` must be one of 'WF93', 'LA08' or 'GFWED'.")
    if method != "WF93" and snd is None:
        raise TypeError(f"Missing input argument snd for fire season method '{method}'.")
    kw = {k: (v if not isinstance(v, tuple) else v[0]) for k, v in default_params.items()}
    kw.update(temp_start_thresh=_param_value("temp_start_thresh", temp_start_thresh),
              temp_end_thresh=_param_value("temp_end_thresh", temp_end_thresh),
              snow_thresh=_param_value("snow_thresh", snow_thresh), temp_condition_days=temp_condition_days,
              snow_condition_days=snow_condition_days)
    affine = [_affine(tas, "degC"), _IDENTITY, _IDENTITY, _IDENTITY,
              _affine(snd, "m") if snd is not None else _IDENTITY]
    series = {"tas": tas, "pr": None, "hurs": None, "ws": None, "snd": None if method == "WF93" else snd}
    state = {"dc0": None, "dmc0": None, "ffmc0": None, "winter_pr": None}
    out = _run(series, affine, None, state, None, ["season_mask"], method, False, None, True, kw)
    return _unitless(out)["season_mask"]


# ------------------------------------------------------------------------------------ element-wise members
def _elementwise(kind, a, b=None, p=(0.0, 0.0, 0.0), attrs=None, scale_b=1.0):
    """Unwrap one or two arrays of any (equal) shape to float32 device tensors, run one element-wise kernel,
    wrap the result like the first labelled argument."""
    import torch
    template = next((x for x in (a, b) if isinstance(x, Field) or is_xarray(x)), None)

    def dev(x):
        if x is None:
            return None
        return device.to_device_f32(raw_values(x) if (isinstance(x, Field) or is_xarray(x)) else x)

    ta, tb = dev(a), dev(b)
    if tb is not None and tuple(tb.shape) != tuple(ta.shape):
        ta, tb = torch.broadcast_tensors(ta, tb)
    if tb is not None and scale_b != 1.0:
        tb = tb * np.float32(scale_b)
    out = device.fire_elementwise(kind, ta, tb, p)
    if template is None:
        return out.cpu().numpy()
    keep_dev = OPTIONS["device_outputs"] and not is_xarray(template)
    vals = out if keep_dev else out.cpu().numpy()
    dims = dims_of(template)
    time = None
    if "time" in dims:
        from .field import time_axis_of
        ta_ = time_axis_of(template)
        time = ta_ if ta_.coord is None else ta_.coord
    return wrap_like(template, vals, tuple(dims), time=time, attrs=dict(attrs or {"units": ""}))


def initial_spread_index(ws, ffmc):
    """Initial spread index from the wind speed [km/h] and the FFMC -- indices/fire/_cffwis.py:449-469."""
    return _elementwise("ISI", ws, ffmc)


def build_up_index(dmc, dc):
    """Build-up index -- indices/fire/_cffwis.py:472-501."""
    return _elementwise("BUI", dmc, dc)


def fire_weather_index(isi, bui):
    """Fire weather index -- indices/fire/_cffwis.py:504-528."""
    return _elementwise("FWI", isi, bui)


def daily_severity_rating(fwi):
    """Daily severity rating -- indices/fire/_cffwis.py:531-546."""
    return _elementwise("DSR", fwi)


def overwintering_drought_code(last_dc, winter_pr, carry_over_fraction=default_params["carry_over_fraction"],
                               wetting_efficiency_fraction=default_params["wetting_efficiency_fraction"],
                               min_dc=default_params["dc_start"]):
    """Season-starting drought code from last season's last DC and the winter precipitation --
    indices/fire/_cffwis.py:1165-1250 (scalar fractions)."""
    if not all(np.isscalar(v) for v in (carry_over_fraction, wetting_efficiency_fraction, min_dc)):
        raise NotImplementedError("overwintering_drought_code: array-valued fractions are not supported")
    scale = 1.0
    if (isinstance(winter_pr, Field) or is_xarray(winter_pr)) and "units" in winter_pr.attrs:
        u = winter_pr.attrs["units"].strip()
        if u not in _LENGTH:
            raise ValueError(f"Cannot convert {u!r} to 'mm'")
        scale = _LENGTH[u] / _LENGTH["mm"]
    return _elementwise("OWDC", last_dc, winter_pr, (carry_over_fraction, wetting_efficiency_fraction, min_dc),
                        scale_b=scale)
