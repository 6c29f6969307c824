"""Standardized indices behind the signatures of ``xclim.indices.stats`` (indices/stats.py:770-1197).

The preprocessing (monthly means, rolling mean), the per-(cell, group) distribution fit and the probability
transform each run as one CUDA kernel over the ``(time, cell)`` buffer; see ``include/xclim_b200.h`` s1.
Supported: ``dist`` in gamma / fisk / lognorm, ``method="APP"`` (any of the three) and ``method="ML"`` with a
fixed ``floc`` (gamma, lognorm), ``freq`` in {"MS", "D", None} on a daily input.
"""
from __future__ import annotations

import json
import warnings

import numpy as np

from . import _lib, device
from .field import attrs_of, dims_of, is_xarray, raw_values, time_axis_of, wrap_like
from .options import OPTIONS

SHAPE_NAMES = {"gamma": "a", "fisk": "c", "lognorm": "s"}
_DIST_METHODS = {"gamma": ["ML", "APP"], "fisk": ["ML", "APP"], "genextreme": ["ML", "APP"], "lognorm": ["ML", "APP"]}


def _check_dist_method(dist, method, fitkwargs):
    """Validation of stats.py:910-936, then what the kernels cover."""
    if method == "APP" and "floc" not in fitkwargs:
        raise ValueError(
            "The APP method is only supported for two-parameter distributions with `gamma`, `fisk`, "
            "`lognorm`, or `genextreme` with `loc` being fixed. Pass a value for `floc` in `fitkwargs`.")
    if not isinstance(dist, str):
        raise NotImplementedError("rv_continuous distribution objects are not supported by the xclim_b200 hot path")
    if dist not in _DIST_METHODS:
        raise NotImplementedError(f"The distribution `{dist}` is not supported.")
    if method not in _DIST_METHODS[dist]:
        raise NotImplementedError(f"The method `{method}` is not supported for distribution `{dist}`.")
    if dist == "genextreme":
        raise NotImplementedError("genextreme is not supported by the xclim_b200 hot path")
    if set(fitkwargs) - {"floc"}:
        raise NotImplementedError(f"fitkwargs {sorted(set(fitkwargs) - {'floc'})} are not supported")
    if method == "ML" and "floc" not in fitkwargs:
        raise NotImplementedError(
            "ML with a free `loc` runs scipy's Nelder-Mead optimiser, whose path depends on last-bit differences of "
            "the likelihood sum; pass `fitkwargs={'floc': ...}` (or use method='APP')")
    if method == "ML" and dist == "fisk":
        raise NotImplementedError("fisk ML has no closed form with a fixed loc: scipy optimises it numerically")


class _Series:
    """The preprocessed series: (T', C) float32 device buffer and its step labels / groups."""

    def __init__(self, y, year, month, day, doy, group, gdim, max_g, calendar, coord):
        self.y, self.year, self.month, self.day, self.doy = y, year, month, day, doy
        self.group, self.gdim, self.max_g, self.calendar, self.coord = group, gdim, max_g, calendar, coord

    def date_key(self):
        return self.year.astype(np.int64) * 10000 + self.month * 100 + self.day

    def labels(self):
        return [f"{int(y):04d}-{int(m):02d}-{int(d):02d}" for y, m, d in zip(self.year, self.month, self.day)]


def _preprocess(da, freq, window, indexer):
    """preprocess_standardized_index (stats.py:770-836): resample, roll, then select_time (NaN steps)."""
    from .timeaxis import TimeAxis
    if freq is not None and freq not in ("MS", "D"):
        if freq.startswith("W"):
            raise NotImplementedError("weekly standardized indices are not supported by the xclim_b200 hot path")
        raise ValueError(f"The input (following resampling if applicable) has a frequency `{freq}` "
                         "which is not supported for standardized indices.")
    if int(window) < 1:
        raise ValueError("window must be >= 1")
    dims = dims_of(da)
    if "time" not in dims:
        raise ValueError("input must have a `time` dimension")
    x2d, cell_shape = device.to_time_cell(raw_values(da), dims.index("time"))
    ta = time_axis_of(da)
    if freq == "MS":
        poff = ta.period_offsets("MS")
        y, _ = device.period_reduce(x2d, poff, _lib.STATS["mean"])
        first = poff[:-1]
        s = _Series(y, ta.year[first], ta.month[first], np.ones(first.size, np.int32), ta.doy[first],
                    ta.month[first] - 1, "month", 12, ta.calendar, None)
        sub = TimeAxis(s.year, s.month, s.day, s.doy, ta.calendar)
    else:
        s = _Series(x2d, ta.year, ta.month, ta.day, ta.doy, ta.doy - 1, "dayofyear", ta.max_doy, ta.calendar,
                    ta.coord)
        sub = ta
    if int(window) > 1:
        s.y = device.rolling_mean(s.y, int(window))
    keep = sub.select_mask(**indexer) if indexer else np.ones(len(s.year), bool)
    return s, keep, cell_shape, tuple(d for d in dims if d != "time")


def _date_bound(s, lo):
    """A "YYYY[-MM[-DD]]" bound as a comparable YYYYMMDD key (start: first day, end: last day of the period)."""
    parts = [int(p) for p in str(s).split("-")]
    y = parts[0]
    m = parts[1] if len(parts) > 1 else (1 if lo else 12)
    d = parts[2] if len(parts) > 2 else (1 if lo else 31)
    return y * 10000 + m * 100 + d


def _cal_slice(series, cal_start, cal_end):
    key = series.date_key()
    lo = 0 if cal_start is None else int(np.searchsorted(key, _date_bound(cal_start, True), side="left"))
    hi = key.size if cal_end is None else int(np.searchsorted(key, _date_bound(cal_end, False), side="right"))
    return slice(lo, max(lo, hi))


def _fit(series, keep, cal, dist, method, zero_inflated, floc):
    """Kernel fit over the calibration steps: (G, 3, C) params, counts, and the groups present in ``cal``."""
    G = series.max_g
    gid = np.asarray(series.group, np.int64)
    idx = np.arange(gid.size)[cal]
    use = idx[keep[cal]]
    order = np.argsort(gid[use], kind="stable")
    steps = use[order]
    goff = np.concatenate([[0], np.cumsum(np.bincount(gid[use], minlength=G))])
    params, nz, nn, status = device.si_fit(series.y, goff, steps, _lib.SI_DISTS[dist], _lib.SI_METHODS[method],
                                           zero_inflated, floc)
    if status & (_lib.SI_STATUS_FITDATA | _lib.SI_STATUS_ROOT_NAN | _lib.SI_STATUS_ROOT_SIGN):
        if status & _lib.SI_STATUS_FITDATA:
            raise ValueError(f"Invalid values in `data`.  Maximum likelihood estimation with '{dist}' requires that "
                             f"{floc!r} < (x - loc)/scale  < inf for each x in `data`.")
        if status & _lib.SI_STATUS_ROOT_NAN:
            raise ValueError("The function value at a bracket end is NaN; solver cannot continue.")
        raise ValueError("f(a) and f(b) must have different signs")
    if status & _lib.SI_STATUS_LOGNORM_FALLBACK:
        raise NotImplementedError("lognorm ML with a fixed loc on a sample of zero spread: scipy falls back to its "
                                  "generic optimiser there")
    present = np.unique(gid[idx])
    return params, nz, nn, present


def _to_host(t, dtype=None):
    if OPTIONS["device_outputs"]:
        return t if dtype is None else t.to(getattr(__import__("torch"), np.dtype(dtype).name))
    a = t.cpu().numpy()
    return a if dtype is None else a.astype(dtype)


def _params_container(da, series, params, nz, nn, present, cell_shape, other, attrs, dist):
    import torch
    gidx = torch.as_tensor(present, device=params.device)
    p = params.index_select(0, gidx).reshape((present.size, 3) + tuple(cell_shape))
    gdim = series.gdim
    groups = present + 1
    coords = {gdim: groups, "dparams": [SHAPE_NAMES[dist], "loc", "scale"]}
    vals = _to_host(p)
    if nz is not None:
        z = _to_host(nz.index_select(0, gidx).reshape((present.size,) + tuple(cell_shape)), np.int64)
        n = _to_host(nn.index_select(0, gidx).reshape((present.size,) + tuple(cell_shape)), np.int64)
        with np.errstate(all="ignore"):
            pz = z / n
        cdims = (gdim,) + tuple(other)
        if is_xarray(da):
            from . import field
            coords.update({k: field.xr.DataArray(np.asarray(v), dims=cdims)
                           for k, v in (("number_of_zeros", z), ("number_of_notnull", n), ("prob_of_zero", pz))})
        else:
            coords.update({"number_of_zeros": z, "number_of_notnull": n, "prob_of_zero": pz})
    return wrap_like(da, vals, (gdim, "dparams") + tuple(other), coords_extra=coords, attrs=attrs)


def standardized_index_fit_params(da, freq, window, dist, method, zero_inflated=False, fitkwargs=None, **indexer):
    """Standardized Index fitting parameters -- indices/stats.py:839-968.  Output dims
    ``(month | dayofyear, dparams, *space)`` float64, dparams in scipy order (shape, loc, scale)."""
    fitkwargs = fitkwargs or {}
    _check_dist_method(dist, method, fitkwargs)
    series, keep, cell_shape, other = _preprocess(da, freq, window, indexer)
    cal = slice(0, len(series.year))
    params, nz, nn, present = _fit(series, keep, cal, dist, method, zero_inflated, float(fitkwargs["floc"]))
    labels = series.labels()
    attrs = {"calibration_period": (labels[0], labels[-1]) if labels else ("", ""), "freq": freq or "",
             "window": window, "scipy_dist": dist, "method": method,
             "group": "time.month" if series.gdim == "month" else "time.dayofyear", "units": "",
             "time_indexer": json.dumps(indexer)}
    return _params_container(da, series, params, nz, nn, present, cell_shape, other, attrs, dist)


def _coord_values(obj, name):
    if is_xarray(obj):
        return np.asarray(obj[name].values) if name in obj.coords else None
    v = obj.coords.get(name)
    if isinstance(v, tuple):
        v = v[1]
    return None if v is None else (v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v))


def _params_on_device(params, series, cell_shape, other, dev):
    """A params array (this module's or real xclim's) -> (G, 3, C) float64 device tensor, counts, groups given."""
    import torch
    gdim = series.gdim
    pdims = dims_of(params)
    if gdim not in pdims:
        raise NotImplementedError(f"params grouped by {pdims[0]!r} do not match the {gdim!r} groups of the data")
    want = (gdim, "dparams") + tuple(other)
    if set(pdims) != set(want):
        raise ValueError(f"params dims {pdims} do not match {want}")
    vals = raw_values(params)
    t = vals.to(dev, torch.float64) if hasattr(vals, "to") else torch.from_numpy(np.asarray(vals, np.float64)).to(dev)
    t = t.permute([pdims.index(d) for d in want]).contiguous()
    groups = np.asarray(_coord_values(params, gdim), np.int64)
    if groups.size and (groups.min() < 1 or groups.max() > series.max_g):
        raise NotImplementedError(f"params {gdim} labels beyond this calendar's {series.max_g} "
                                  "(params from another calendar)")
    # a day-of-year table that ends on the last day of a 360-, 365- or 366-day year other than the data's comes
    # from another calendar: the reference converts it (resample_doy), this path would pair days wrongly
    if gdim == "dayofyear" and groups.size and int(groups.max()) in (360, 365, 366) and \
            int(groups.max()) != series.max_g:
        raise NotImplementedError(f"day-of-year params of a {int(groups.max())}-day calendar on data of a "
                                  f"{series.max_g}-day calendar (params from another calendar) are not supported")
    G = series.max_g
    C = int(np.prod(cell_shape)) if cell_shape else 1
    full = torch.full((G, 3, C), float("nan"), dtype=torch.float64, device=dev)
    gi = torch.as_tensor(groups - 1, device=dev)
    full.index_copy_(0, gi, t.reshape(groups.size, 3, C))
    counts = []
    for name in ("number_of_zeros", "number_of_notnull"):
        v = _coord_values(params, name)
        if v is None:
            counts.append(None)
            continue
        cdims = (gdim,) + tuple(other)
        if is_xarray(params) and tuple(params[name].dims) != cdims:
            v = np.asarray(params[name].transpose(*cdims).values)
        cz = torch.zeros((G, C), dtype=torch.int32, device=dev)
        cz.index_copy_(0, gi, torch.from_numpy(np.ascontiguousarray(v, np.int64).astype(np.int32)).to(dev)
                       .reshape(groups.size, C))
        counts.append(cz)
    return full, counts[0], counts[1], groups - 1


def standardized_index(da, freq, window, dist, method, zero_inflated, fitkwargs, cal_start, cal_end, params=None,
                       prob_zero_interpolation="upper", plotting_position_zero="ecdf", **indexer):
    """Standardized Index -- indices/stats.py:971-1197.  float64 ``(time, *space)`` on the resampled axis."""
    if params is None and None in [window, dist, method, zero_inflated]:
        raise ValueError("If `params` is `None`, `window`, `dist`, `method` and `zero_inflated` must be given.")
    if params is not None:
        pa = attrs_of(params)
        freq, window, dist, indexer = (pa[s] for s in ["freq", "window", "scipy_dist", "time_indexer"])
        freq = None if freq == "" else freq
        indexer = json.loads(indexer)
        if cal_start or cal_end:
            warnings.warn("Expected either `cal_{start|end}` or `params`, got both. The `params` input overrides "
                          "other inputs.If `cal_start`, `cal_end`, `freq`, `window`, and/or `dist` were given as "
                          "input, they will be ignored.")
        zero_inflated = any(k in pa for k in ["number_of_zeros", "prob_of_zero"])
    if zero_inflated is not None:
        interp = {"center": 1 / 2, "upper": 1}.get(prob_zero_interpolation, None)
        if interp is None:
            if isinstance(prob_zero_interpolation, str):
                raise ValueError("Accepted strings for `prob_zero_interpolation` are: ['center', 'upper']")
            interp = prob_zero_interpolation
        alpha_beta = {"ecdf": (0, 1), "weibull": (0, 0)}.get(plotting_position_zero, None)
        if alpha_beta is None:
            if isinstance(plotting_position_zero, str):
                raise ValueError("Accepted strings for `plotting_position_zero` are: ['ecdf', 'weibull']")
            alpha_beta = plotting_position_zero
    if params is None:
        fitkwargs = fitkwargs or {}
        _check_dist_method(dist, method, fitkwargs)
    elif dist not in SHAPE_NAMES:
        raise NotImplementedError(f"params of the `{dist}` distribution are not supported by the xclim_b200 hot path")
    series, keep, cell_shape, other = _preprocess(da, freq, window, indexer)
    gid = np.asarray(series.group, np.int64)
    if params is None:
        cal = _cal_slice(series, cal_start, cal_end)
        pdev, nz, nn, present = _fit(series, keep, cal, dist, method, zero_inflated, float(fitkwargs["floc"]))
        if not zero_inflated:
            nz = nn = None
        pattrs = {"calibration_period": None, "freq": "", "window": 1, "scipy_dist": dist, "method": method,
                  "group": "time.month" if series.gdim == "month" else "time.dayofyear", "units": "",
                  "time_indexer": "{}"}
    else:
        if _coord_values(params, "prob_of_zero") is not None and _coord_values(params, "number_of_zeros") is None:
            raise NotImplementedError("params carrying only `prob_of_zero` (an old xclim version) are not supported")
        pdev, nz, nn, present = _params_on_device(params, series, cell_shape, other, series.y.device)
        pattrs = dict(attrs_of(params))
    gos = np.where(keep & np.isin(gid, present), gid, -1)
    a, b = alpha_beta
    out = device.si_apply(series.y, gos, pdev, nz, nn, _lib.SI_DISTS[dist], float(interp), float(a), float(b))
    vals = out.reshape((out.shape[0],) + tuple(cell_shape))
    vals = vals if (OPTIONS["device_outputs"] and not is_xarray(da)) else vals.cpu().numpy()
    attrs = dict(pattrs)
    if attrs.get("calibration_period") is None:
        lab = series.labels()[_cal_slice(series, cal_start, cal_end)]
        attrs["calibration_period"] = (lab[0], lab[-1]) if lab else ("", "")
    attrs["freq"] = freq or "D"
    attrs["window"] = window
    attrs["units"] = ""
    time = series.coord if series.coord is not None else np.array(series.labels())
    if series.gdim == "month":
        from .generic import _period_time
        time = _period_time(da, time_axis_of(da), "MS")
    if not is_xarray(da) and series.gdim == "dayofyear":
        time = time_axis_of(da)
    return wrap_like(da, vals, ("time",) + tuple(other), time=time, attrs=attrs)


# ------------------------------------------------------------------------ frequency analysis (stats.py:115-548)
_FIT_METHOD_NAMES = {"ML": "maximum likelihood", "MM": "method of moments", "MLE": "maximum likelihood",
                     "MSE": "maximum product of spacings", "MPS": "maximum product of spacings",
                     "PWM": "probability weighted moments", "APP": "approximative method"}
_EV_PARAM_NAMES = {"norm": ["loc", "scale"], "gumbel_r": ["loc", "scale"], "genextreme": ["c", "loc", "scale"]}


def _ev_dist(dist):
    """get_dist (stats.py:551-573) for the laws the frequency-analysis kernels cover."""
    if not isinstance(dist, str):
        raise NotImplementedError("rv_continuous distribution objects are not supported by the xclim_b200 hot path")
    if dist in _EV_PARAM_NAMES:
        return dist
    try:
        import scipy.stats
        known = getattr(scipy.stats, dist, None) is not None
    except ImportError:     # pragma: no cover - scipy only tells an unknown name from an unsupported one
        known = True
    if not known:
        raise ValueError(f"Statistical distribution `{dist}` is not found in scipy.stats.")
    raise NotImplementedError(f"The distribution `{dist}` is not supported by the xclim_b200 frequency analysis "
                              f"(supported: {', '.join(_EV_PARAM_NAMES)}).")


def _prefix_attrs(attrs, names, prefix):
    return {(prefix + k if k in names else k): v for k, v in attrs.items()}


def _unprefix_attrs(attrs, names, prefix):
    """xclim.core.formatting.unprefix_attrs: a prefixed key wins over the plain one."""
    out = {}
    for k, v in attrs.items():
        if k.startswith(prefix) and k[len(prefix):] in names:
            out[k[len(prefix):]] = v
        elif k not in out:
            out[k] = v
    return out


def _history(text, name):
    from datetime import datetime
    return f"[{datetime.now().strftime('%Y-%m-%d %H:%M:%S')}] {name}: {text} - xclim_b200"


def _output(template, out_dev, lead_dims_shape, dims, coords, attrs):
    vals = out_dev.reshape(lead_dims_shape)
    vals = vals if (OPTIONS["device_outputs"] and not is_xarray(template)) else vals.cpu().numpy()
    return wrap_like(template, vals, dims, coords_extra=coords, attrs=attrs)


def fit(da, dist="norm", method="ML", dim="time", **fitkwargs):
    """Fit a univariate law along time, per cell -- indices/stats.py:115-218.  float64, ``dparams`` in place of
    ``time``, coordinates in scipy's order.  Maximum likelihood (``ML`` / ``MLE``) of ``norm``, ``gumbel_r`` and
    ``genextreme`` (xc_ev_fit_f32); NaN and +-inf values are dropped, a cell with <= 1 value left is NaN."""
    method = method.upper()
    if method not in _FIT_METHOD_NAMES:
        raise ValueError(f"Fitting method not recognized: {method}")
    dist = _ev_dist(dist)
    if method == "PWM":
        raise ValueError(f"The given distribution {dist} does not implement the PWM fitting method. "
                         "Please pass an instance from the lmoments3 package.")
    if method not in ("ML", "MLE"):
        why = {"MM": "scipy runs its generic moment-matching optimiser there",
               "APP": "the approximative method has no start values for these laws",
               "MSE": "scipy.stats.fit's spacing optimiser is not reproduced",
               "MPS": "scipy.stats.fit's spacing optimiser is not reproduced"}[method]
        raise NotImplementedError(f"method {method!r} is not supported by the xclim_b200 frequency analysis: {why}")
    if dim != "time":
        raise NotImplementedError(f"fits along {dim!r} are not supported: the kernels fit along `time`")
    if fitkwargs:
        raise NotImplementedError(f"fitkwargs {sorted(fitkwargs)} (fixed parameters, optimiser options) are not "
                                  "supported by the xclim_b200 frequency analysis")
    dims = dims_of(da)
    if "time" not in dims:
        raise ValueError("input must have a `time` dimension")
    x2d, cell_shape = device.to_time_cell(raw_values(da), dims.index("time"))
    params, status = device.ev_fit(x2d, _lib.EV_DISTS[dist])
    if status & _lib.EV_STATUS_ROOT_NAN:
        raise ValueError("The function value at a bracket end is NaN; solver cannot continue.")
    if status & _lib.EV_STATUS_ROOT_SIGN:
        raise ValueError("f(a) and f(b) must have different signs")
    if status & (_lib.EV_STATUS_NOT_CONVERGED | _lib.EV_STATUS_UNBOUNDED):
        import torch
        fitted = torch.isfinite(x2d).sum(0) > 1
        bad = int((fitted & torch.isnan(params[0])).sum().item())
        why = "the likelihood has no maximum (c >= 1) or the Newton iterations did not converge"
        warnings.warn(f"{dist} fit: {bad} cell(s) set to NaN: {why}", RuntimeWarning)
    names = _EV_PARAM_NAMES[dist]
    ti = dims.index("time")
    out = params.reshape((len(names),) + tuple(cell_shape))
    out = out.permute(*([k for k in range(1, ti + 1)] + [0] + [k for k in range(ti + 1, len(dims))]))
    out_dims = tuple(d if d != "time" else "dparams" for d in dims)
    attrs = _prefix_attrs(attrs_of(da), ["standard_name", "long_name", "units", "description"], "original_")
    attrs.update({"long_name": f"{dist} parameters", "description": f"Parameters of the {dist} distribution",
                  "method": method, "estimator": _FIT_METHOD_NAMES[method].capitalize(), "scipy_dist": dist,
                  "units": "",
                  "history": _history(f"Estimate distribution parameters by {_FIT_METHOD_NAMES[method]} method "
                                      f"along dimension {dim}.", "fit")})
    return _output(da, out.contiguous(), tuple(out.shape), out_dims, {"dparams": names}, attrs)


def _params_2d(p, dist):
    """A fitted-parameters array -> ((P, C) float64 tensor, its dims, dparams position, cell shape)."""
    import torch
    dims = dims_of(p)
    if "dparams" not in dims:
        raise ValueError("the parameters need a `dparams` dimension")
    vals = raw_values(p)
    t = vals if isinstance(vals, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(vals, np.float64))
    t = t.to(torch.float64)
    k = dims.index("dparams")
    if t.shape[k] != len(_EV_PARAM_NAMES[dist]):
        raise ValueError(f"{dist} has {len(_EV_PARAM_NAMES[dist])} parameters, `dparams` has {t.shape[k]}")
    t = t.movedim(k, 0).contiguous()
    rest = tuple(t.shape[1:])
    return t.reshape(t.shape[0], -1), dims, k, rest


def _transformed(p, dist, kind, q, new_dim, coord, attrs):
    params, dims, k, rest = _params_2d(p, dist)
    if params.shape[1] == 0:
        import torch
        out = torch.empty((len(q), 0), dtype=torch.float64, device=params.device)
    else:
        out = device.ev_transform(params, _lib.EV_DISTS[dist], _lib.EV_KINDS[kind], q)
    out = out.reshape((len(q),) + rest).movedim(0, k).contiguous()
    out_dims = tuple(d if d != "dparams" else new_dim for d in dims)
    return _output(p, out, tuple(out.shape), out_dims, {new_dim: coord}, attrs)


def _quantiles(p, q, dist, new_dim, coord):
    dist = _ev_dist(dist or attrs_of(p)["scipy_dist"])
    attrs = _unprefix_attrs(attrs_of(p), ["units", "standard_name"], "original_")
    attrs.update({"long_name": f"{dist} quantiles", "description": f"Quantiles estimated by the {dist} distribution",
                  "cell_methods": "dparams: ppf",
                  "history": _history("Compute parametric quantiles from distribution parameters",
                                      "parametric_quantile")})
    if np.all(q > 0.5):
        return _transformed(p, dist, "isf", 1 - q, new_dim, coord, attrs)
    return _transformed(p, dist, "ppf", q, new_dim, coord, attrs)


def parametric_quantile(p, q, dist=None):
    """Quantiles of the fitted laws -- indices/stats.py:221-289: ``isf(1 - q)`` when every q > 0.5, else
    ``ppf(q)``; ``dparams`` becomes ``quantile`` (xc_ev_transform_f64)."""
    q = np.atleast_1d(q)
    return _quantiles(p, q, dist, "quantile", q)


def parametric_cdf(p, v, dist=None):
    """CDF of the fitted laws at the values ``v`` -- indices/stats.py:294-360; ``dparams`` becomes ``cdf``."""
    if hasattr(v, "dims"):
        if len(v.dims) > 1:
            raise ValueError("`v` must be one-dimensional.")
        v = np.asarray(v.values)
    v = np.atleast_1d(v)
    dist = _ev_dist(dist or attrs_of(p)["scipy_dist"])
    attrs = _unprefix_attrs(attrs_of(p), ["units", "standard_name"], "original_")
    attrs.update({"long_name": f"{dist} cdf", "description": f"CDF estimated by the {dist} distribution",
                  "cell_methods": "dparams: cdf",
                  "history": _history("Compute parametric cdf from distribution parameters", "parametric_cdf")})
    return _transformed(p, dist, "cdf", np.asarray(v, np.float64), "cdf", v, attrs)


def fa(da, t, dist="norm", mode="max", method="ML"):
    """Return levels -- indices/stats.py:429-475: the value of return period ``t`` (exceedance for ``mode``
    max / high, non-exceedance for min / low); output dim ``return_period``."""
    p = fit(da, dist, method=method)
    t = np.atleast_1d(t)
    if mode in ["max", "high"]:
        q = 1 - 1.0 / t
    elif mode in ["min", "low"]:
        q = 1.0 / t
    else:
        raise ValueError(f"Mode `{mode}` should be either 'max' or 'min'.")
    out = _quantiles(p, q, dist, "return_period", t)
    out.attrs["mode"] = mode
    return out


def _extremes(da, mode, window, freq, **indexer):
    """The per-period extremes of frequency_analysis (stats.py:526-538): rolling mean (skipna=False), then
    select_resample_op(op=mode) with the indexer."""
    from . import generic
    from .units import to_agg_units_attrs
    dims = dims_of(da)
    if "time" not in dims:
        raise ValueError("input must have a `time` dimension")
    x2d, cell_shape = device.to_time_cell(raw_values(da), dims.index("time"))
    other = tuple(d for d in dims if d != "time")
    ta = time_axis_of(da)
    if int(window) > 1:
        x2d = device.rolling_mean(x2d, int(window))
    if indexer:
        keep = ta.select_mask(**indexer)
        if not keep.all():
            x2d = device.mask_steps(x2d, keep)
    out, _ = device.period_reduce(x2d, ta.period_offsets(freq), _lib.STATS[mode])
    attrs = attrs_of(da)
    attrs.update(to_agg_units_attrs(da, mode))
    return generic._wrap_periods(da, out, tuple(cell_shape), other, ta, freq, attrs)


def frequency_analysis(da, mode, t, dist, window=1, freq=None, method="ML", **indexer):
    """Return levels of the per-period extremes -- indices/stats.py:478-548.  Host-backed inputs stream through
    HBM in slabs for the extremes (xclim_b200/streaming.py); only the (periods, cells) extremes are fitted."""
    from . import generic
    from .streaming import streamed
    if mode not in ("max", "min"):
        raise ValueError(f"Mode `{mode}` should be either 'max' or 'min'.")
    freq = freq or generic.default_freq(**indexer)
    sel = streamed(_extremes)(da, mode, window, freq, **indexer)
    return fa(sel, t, dist=dist, mode=mode, method=method)
