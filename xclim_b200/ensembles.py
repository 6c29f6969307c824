"""Ensemble statistics behind the signatures of ``xclim.ensembles`` (ensembles/_base.py, ensembles/_robustness.py).

The reductions across realizations run as CUDA kernels over the ``(realization, cell)`` matrix (include/xclim_b200.h
e1): ``ensemble_percentiles`` and ``ensemble_mean_std_max_min`` one lane per cell, ``robustness_fractions`` one lane
per cell walking every member's series.  Inputs are ``Field``s or DataArrays with a ``realization`` dim in any
position; ``create_ensemble`` stacks aligned members (on the device when they are device-resident).  Host-backed
inputs of at least ``stream_min_bytes`` are walked in column ranges of about ``stream_slab_bytes`` for the
percentiles and moments; ``robustness_fractions`` stages its inputs to the device whole.
"""
from __future__ import annotations

import os

import numpy as np

from . import _lib, device
from . import field as _field
from .field import Field, is_xarray
from .options import OPTIONS

REALIZATION = "realization"

# ensembles/_base.py:21-28
_quantile_params = {
    "interpolated_inverted_cdf": (0, 1),
    "hazen": (0.5, 0.5),
    "weibull": (0, 0),
    "linear": (1, 1),
    "median_unbiased": (1 / 3, 1 / 3),
    "normal_unbiased": (3 / 8, 3 / 8),
}

SIGNIFICANCE_TESTS = ("ttest", "welch-ttest", "mannwhitney-utest", "brownforsythe-test", "ipcc-ar6-c")
_UNSUPPORTED_TESTS = {
    "mannwhitney-utest": "scipy switches between its exact and asymptotic U distributions by sample size and ties",
    "brownforsythe-test": "the Brown-Forsythe test has no device kernel",
}

#: device on which host columns are staged (the CPU tests substitute their stand-ins)
_DEVICE = "cuda"


# ------------------------------------------------------------------------------------------ containers
def _is_dataset(obj) -> bool:
    return _field.xr is not None and hasattr(_field.xr, "Dataset") and isinstance(obj, _field.xr.Dataset)


def _variables(ens) -> dict:
    """The variables of a Dataset (or a dict of members standing in for one), or {name: ens} for one array."""
    if _is_dataset(ens):
        return dict(ens.data_vars)
    if isinstance(ens, dict):
        return dict(ens)
    return {ens.name: ens}


def _collect(parts: dict, template):
    """Several named outputs: an xr.Dataset for xarray inputs where xarray has one, else a dict."""
    if is_xarray(template) and hasattr(_field.xr, "Dataset"):
        return _field.xr.Dataset(parts)
    return parts


def _wrap(template, values, dims, attrs, name, coords_extra=None):
    keep_dev = OPTIONS["device_outputs"] and not is_xarray(template)
    if hasattr(values, "is_cuda") and not keep_dev:
        values = values.cpu().numpy()
    coords = {d: template.coords[d] for d in dims if d in getattr(template, "coords", {})}
    coords.update(coords_extra or {})
    if is_xarray(template):
        return _field.xr.DataArray(values, dims=dims, coords=coords, attrs=attrs, name=name)
    time = template.time if "time" in dims else None
    return Field(values, tuple(dims), time, coords, attrs, name)


def _realization_axis(da) -> int:
    dims = tuple(da.dims)
    if REALIZATION not in dims:
        raise ValueError(f"the input has no `{REALIZATION}` dimension: {dims}")
    return dims.index(REALIZATION)


def _n_members(ens) -> int:
    da = next(iter(_variables(ens).values()))
    return int(da.shape[_realization_axis(da)])


# ------------------------------------------------------------------------------------------ create
def create_ensemble(datasets, multifile=False, resample_freq=None, calendar=None, realizations=None, cal_kwargs=None,
                    **xr_kwargs):
    """Stack already aligned members along a new leading ``realization`` dim (ensembles/_base.py:31-138).

    ``datasets``: a list (or dict keyed by realization) of Fields or DataArrays with identical dims, shape and
    time axis.  Device-resident members are stacked on the device.  Opening files, time alignment,
    ``resample_freq`` and calendar conversion are not supported.  Returns a Field for Fields, an xr.Dataset for
    DataArrays (as the reference)."""
    if multifile or resample_freq is not None or calendar is not None or cal_kwargs or xr_kwargs:
        raise NotImplementedError("create_ensemble only stacks aligned members: no file options, `resample_freq`, "
                                  "`calendar` or time alignment")
    if isinstance(datasets, dict):
        if realizations is None:
            realizations, datasets = list(datasets.keys()), list(datasets.values())
        else:
            datasets = list(datasets.values())
    if isinstance(datasets, (str, os.PathLike)):
        raise NotImplementedError("paths and glob patterns are not supported: pass the members themselves")
    members = list(datasets)
    if not members:
        raise ValueError("create_ensemble needs at least one member")
    for m in members:
        if isinstance(m, (str, os.PathLike, list, tuple)):
            raise NotImplementedError("paths and glob patterns are not supported: pass the members themselves")
        if not (isinstance(m, Field) or is_xarray(m)):
            raise NotImplementedError(f"members must be Fields or DataArrays, got {type(m).__name__}")
    first = members[0]
    if any(isinstance(m, Field) != isinstance(first, Field) for m in members):
        raise ValueError("members must all be Fields or all DataArrays")
    for i, m in enumerate(members[1:], 1):
        if tuple(m.dims) != tuple(first.dims) or tuple(m.shape) != tuple(first.shape):
            raise NotImplementedError(f"member #{i:02d} has dims {tuple(m.dims)} and shape {tuple(m.shape)}, not "
                                      f"{tuple(first.dims)} {tuple(first.shape)}: aligning members is not supported")
        if "time" in first.dims and not _same_time(first, m):
            raise NotImplementedError(f"member #{i:02d} has another time axis: aligning members is not supported")
    if realizations is None:
        realizations = np.arange(len(members))
    vals = [m.values for m in members]
    if all(hasattr(v, "is_cuda") and v.is_cuda for v in vals):
        import torch
        stacked = torch.stack(vals)
    else:
        stacked = np.stack([v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v) for v in vals])
    dims = (REALIZATION,) + tuple(first.dims)
    coords = {REALIZATION: np.asarray(list(realizations))}
    if isinstance(first, Field):
        return Field(stacked, dims, first.time, {**first.coords, **coords}, dict(first.attrs), first.name)
    crd = {d: first.coords[d] for d in first.dims if d in first.coords}
    da = _field.xr.DataArray(stacked, dims=dims, coords={**crd, **coords}, attrs=dict(first.attrs), name=first.name)
    return _field.xr.Dataset({first.name: da}) if hasattr(_field.xr, "Dataset") else da


def _same_time(a, b) -> bool:
    if isinstance(a, Field):
        ta, tb = a.time, b.time
        if ta is None or tb is None:
            return ta is tb
        return ta.calendar == tb.calendar and all(np.array_equal(getattr(ta, k), getattr(tb, k))
                                                  for k in ("year", "month", "day"))
    return np.array_equal(np.asarray(a.coords["time"].values), np.asarray(b.coords["time"].values))


# ------------------------------------------------------------------------------------------ column walk
def _column_reduce(da, fn):
    """Apply ``fn((R, w) float32 device matrix) -> list of (k, w) or (w,) tensors`` over the columns of
    ``da`` (realization moved first).  Returns the results as (k, N) / (N,) tensors, or numpy arrays when
    the input was host-backed and walked in column ranges, and the shape of the non-member dims."""
    import torch
    ax = _realization_axis(da)
    v = da.values
    R = int(v.shape[ax])
    rest = tuple(s for i, s in enumerate(v.shape) if i != ax)
    N = int(np.prod(rest, dtype=np.int64))
    if hasattr(v, "is_cuda") and v.is_cuda:
        x = v.movedim(ax, 0).to(torch.float32).reshape(R, N)
        return fn(x if x.stride(1) == 1 else x.contiguous()), rest
    a = np.moveaxis(np.asarray(v), ax, 0)
    a = np.ascontiguousarray(a, dtype=np.float32).reshape(R, N)
    if a.nbytes < OPTIONS["stream_min_bytes"]:
        return fn(torch.from_numpy(a).to(_DEVICE)), rest
    # host-backed and large: one strided box of R rows per column range, results copied back range by range
    lib = _lib.load()
    w = int(max(1, min(N, OPTIONS["stream_slab_bytes"] // (4 * R))))
    buf = torch.empty((R, w), dtype=torch.float32, device=_DEVICE)
    outs = None
    for n0 in range(0, N, w):
        n1 = min(N, n0 + w)
        x = buf[:, :n1 - n0]
        _lib.check(lib.xc_copy_box_async(buf.data_ptr(), 4 * w, a.ctypes.data + 4 * n0, 4 * N, 4 * (n1 - n0), R, 1,
                                         device.current_stream_ptr()))
        res = fn(x)
        if outs is None:
            outs = [np.empty(r.shape[:-1] + (N,), dtype=str(r.dtype).replace("torch.", "")) for r in res]
        for o, r in zip(outs, res):
            o[..., n0:n1] = r.cpu().numpy()
    return outs, rest


# ------------------------------------------------------------------------------------------ percentiles
def ensemble_percentiles(ens, values=None, keep_chunk_size=None, min_members=1, weights=None, split=True,
                         method="linear"):
    """Percentiles across realizations (ensembles/_base.py:214-373).  ``keep_chunk_size`` (dask advice) is ignored.

    Float64 results for two or more members, the input's float32 for one (``calc_perc``'s dtypes)."""
    if values is None:
        values = [10, 50, 90]
    if weights is not None:
        raise NotImplementedError("weighted ensemble percentiles use xarray's weighted quantile, a different "
                                  "algorithm: not supported")
    if method not in _quantile_params:
        raise ValueError(f"method must be one of {list(_quantile_params)}, got {method!r}")
    if min_members is None:
        min_members = _n_members(ens)
    if _is_dataset(ens) or isinstance(ens, dict):
        parts = {}
        template = None
        for da in _variables(ens).values():
            if REALIZATION in tuple(da.dims):
                template = da
                res = ensemble_percentiles(da, values, min_members=min_members, split=split, method=method)
                parts.update(_variables(res) if (split or _is_dataset(res)) else {da.name: res})
        out = _collect(parts, template)
        if _is_dataset(ens):
            out.attrs.update(ens.attrs)
        return out
    alpha, beta = _quantile_params[method]
    per = [float(p) for p in values]
    res, rest = _column_reduce(ens, lambda x: [device.ens_percentiles(x, per, alpha, beta, min_members)])
    vals = res[0].reshape((len(per),) + rest)
    rest_dims = tuple(d for d in ens.dims if d != REALIZATION)
    attrs = dict(ens.attrs)
    if not split:
        moved = vals.movedim(0, -1).contiguous() if hasattr(vals, "movedim") else np.moveaxis(vals, 0, -1)
        return _wrap(ens, moved, rest_dims + ("percentiles",), attrs, ens.name,
                     {"percentiles": np.asarray(list(values))})
    parts = {}
    for k, p in enumerate(values):
        a = dict(attrs)
        a["description"] = a.get("description", "") + f" {p}th percentile of ensemble."
        name = f"{ens.name}_p{int(p):02d}"
        parts[name] = _wrap(ens, vals[k], rest_dims, a, name)
    return _collect(parts, ens)


# ------------------------------------------------------------------------------------------ moments
def _weights_array(weights, R):
    if weights is None:
        return None
    w = weights.values if hasattr(weights, "dims") else weights
    w = w.detach().cpu().numpy() if hasattr(w, "detach") else np.asarray(w)
    w = np.asarray(w, dtype=np.float64).ravel()
    if np.isnan(w).any():
        raise ValueError("`weights` cannot contain missing values. Missing values can be replaced by "
                         "`weights.fillna(0)`.")
    if w.size != R:
        raise ValueError(f"weights have {w.size} values for {R} realizations")
    return w


def ensemble_mean_std_max_min(ens, min_members=1, weights=None):
    """Mean, standard deviation (ddof 0), maximum and minimum across realizations (ensembles/_base.py:141-211):
    ``{v}_mean``, ``{v}_stdev``, ``{v}_max``, ``{v}_min`` for each variable.  Unweighted: float32 (float64 sums
    rounded once); weighted: float64 mean / stdev with xarray's Weighted formulas."""
    import torch
    R = _n_members(ens)
    if min_members is None:
        min_members = R
    w = _weights_array(weights, R)
    parts, template = {}, None
    for v, da in _variables(ens).items():
        template = da
        wd = None if w is None else torch.from_numpy(w).to(da.values.device if hasattr(da.values, "is_cuda")
                                                              else _DEVICE)
        res, rest = _column_reduce(da, lambda x: list(device.ens_moments(x, wd, min_members)))
        rest_dims = tuple(d for d in da.dims if d != REALIZATION)
        for stat, val in zip(("mean", "stdev", "max", "min"), (res[0], res[1], res[3], res[2])):
            name = f"{v}_{stat}"
            attrs = dict(da.attrs)
            if "description" in attrs:     # _base.py:205, word for word ("tg_mean" -> "mean_mean of ensemble")
                attrs["description"] = attrs["description"] + " : " + name.split("_", maxsplit=1)[-1] + " of ensemble"
            parts[name] = _wrap(da, val.reshape(rest), rest_dims, attrs, name)
    out = _collect(parts, template)
    if _is_dataset(ens):
        out.attrs.update(ens.attrs)
    return out


# ------------------------------------------------------------------------------------------ robustness
def _member_series(da, with_time):
    """(R, T, C) float32 device tensor with unit cell stride, the non-member, non-time dims, their shape and the
    dims of ``da`` without time (a dummy realization first when ``da`` has none)."""
    import torch
    dims = list(da.dims)
    v = da.values
    if REALIZATION not in dims:                        # a dummy realization (_robustness.py:200-206)
        dims = [REALIZATION] + dims
        v = v[None] if hasattr(v, "is_cuda") else np.asarray(v)[None]
    if not with_time and "time" in dims:
        raise ValueError("When deltas are given (ref=None), `fut` holds one delta per member and cell: it must not "
                         "have a `time` dimension.")
    order = [dims.index(REALIZATION)] + ([dims.index("time")] if with_time else [])
    rest_dims = tuple(d for d in dims if d not in (REALIZATION, "time"))
    order += [dims.index(d) for d in rest_dims]
    t = v if hasattr(v, "is_cuda") else torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32))
    t = t.permute(order).to(device=_DEVICE if not getattr(t, "is_cuda", False) else t.device, dtype=torch.float32)
    R = t.shape[0]
    T = t.shape[1] if with_time else 1
    rest = tuple(t.shape[2 if with_time else 1:])
    t = t.reshape(R, T, -1)
    if t.stride(2) != 1:
        t = t.contiguous()
    return t, rest_dims, rest, tuple(d for d in dims if d != "time")


def _ys_annual_means(ref, r3):
    """The YS means of every member of ``ref`` (R, P, C) float32 (the period_reduce kernel) and the YS timestamps
    (P) float64 in days since the first: `ref.resample(time="YS").mean()` of _robustness.py:651."""
    import torch

    from .field import time_axis_of
    from .timeaxis import _is_leap
    ta = time_axis_of(ref)
    if len(ta) != r3.shape[1]:
        raise ValueError("the time axis of `ref` does not match its data")
    poff = ta.period_offsets("YS")
    refy = torch.stack([device.period_reduce(r3[r], poff, _lib.STATS["mean"])[0] for r in range(r3.shape[0])])
    years = np.asarray(ta.year)[poff[:-1]].astype(np.int64)
    span = np.arange(years[0], years[-1] + 1)
    ndays = np.full(span.size, 360) if ta.calendar == "360_day" else 365 + _is_leap(span, ta.calendar).astype(int)
    start = np.concatenate([[0], np.cumsum(ndays)[:-1]])          # Jan 1 of each year, days after the first
    ys = torch.from_numpy(start[years - years[0]].astype(np.float64)).to(r3.device)
    return refy, ys


def _check_invalid(invalid):
    if invalid is None:
        return
    if getattr(invalid, "__name__", None) == "missing_any" or type(invalid).__name__ == "MissingAny":
        return
    raise NotImplementedError("only MissingAny (a member is invalid where any time step of fut or ref is NaN) is "
                              "supported as `invalid`")


def robustness_fractions(fut, ref=None, test=None, weights=None, invalid=None, strict_sign=True, **kwargs):
    """Fractions of members showing significant change and agreeing on its sign (ensembles/_robustness.py:74-333).

    Returns ``changed``, ``positive``, ``changed_positive``, ``negative``, ``changed_negative``, ``valid``,
    ``agree`` (float64, no ``realization`` or ``time`` dim) and, for the t-tests, ``pvals`` (float32, with the
    ``realization`` dim, in ``fut``'s dim order); as an xr.Dataset for DataArrays, a dict of Fields for Fields.
    Tests: None, "threshold", "ttest", "welch-ttest" and "ipcc-ar6-c" without ``ref_pi`` (``ref`` needs its time
    axis); the statistics are float64 (DESIGN.md section 4)."""
    if ref is None:
        if test not in [None, "threshold"]:
            raise ValueError("When deltas are given (ref=None), 'test' must be None or 'threshold'.")
    else:
        _check_invalid(invalid)
    param, test_params = 0.0, {}
    if test is None:
        code = _lib.ENS_TESTS[None]
    elif test == "threshold":
        abs_thresh, rel_thresh = kwargs.get("abs_thresh"), kwargs.get("rel_thresh")
        if abs_thresh is not None and rel_thresh is None:
            code, param, test_params = _lib.ENS_TESTS["abs_thresh"], float(abs_thresh), {"abs_thresh": abs_thresh}
        elif rel_thresh is not None and abs_thresh is None:
            if ref is None:
                raise ValueError("`rel_thresh` divides by the mean of `ref`: it needs `ref`")
            code, param, test_params = _lib.ENS_TESTS["rel_thresh"], float(rel_thresh), {"rel_thresh": rel_thresh}
        else:
            raise ValueError("One and only one of abs_thresh or rel_thresh must be given if test='threshold'.")
    elif test in _UNSUPPORTED_TESTS:
        raise NotImplementedError(f"test {test!r} is not supported: {_UNSUPPORTED_TESTS[test]}")
    elif test == "ipcc-ar6-c":
        if kwargs.get("ref_pi") is not None:
            raise NotImplementedError("ipcc-ar6-c with `ref_pi` (20-year means of quadratically detrended "
                                      "pre-industrial data) is not supported")
        code, test_params = _lib.ENS_TESTS[test], {"ref_pi": None}
    elif test in SIGNIFICANCE_TESTS:
        code = _lib.ENS_TESTS[test]
        test_params = {"p_change": kwargs.get("p_change", 0.05)}
        param = float(test_params["p_change"])
    else:
        raise ValueError(f"Statistical test {test} must be one of {', '.join(SIGNIFICANCE_TESTS)}.")
    import torch
    f3, rest_dims, rest, p_dims = _member_series(fut, ref is not None)
    r3 = _member_series(ref, True)[0] if ref is not None else None
    R = f3.shape[0]
    if r3 is not None and (r3.shape[0] != R or r3.shape[2] != f3.shape[2]):
        raise ValueError("`fut` and `ref` must have the same realizations and cells")
    w = _weights_array(weights, R)
    wd = None if w is None else torch.from_numpy(w).to(f3.device)
    want_p = test in ("ttest", "welch-ttest")
    refy, ys = _ys_annual_means(ref, r3) if test == "ipcc-ar6-c" else (None, None)
    frac, pvals = device.ens_robustness(f3, r3, wd, code, param, strict_sign, want_p, refy, ys)
    kw = ", ".join(f"{k}={v}" for k, v in test_params.items())
    test_str = f"Significant change was tested with test {test} and parameters {kw}."
    strict = "strictly " if strict_sign else "zero or "
    desc = {
        "changed": (f"Fraction of valid members showing significant change. {test_str}", True),
        "positive": (f"Fraction of valid members showing {strict} positive change.", False),
        "changed_positive": (f"Fraction of valid members showing significant and {strict} positive change. "
                             f"{test_str}", True),
        "negative": (f"Fraction of valid members showing {strict} negative change.", False),
        "changed_negative": (f"Fraction of valid members showing significant and {strict} negative change. "
                             f"{test_str}", True),
        "valid": ("Fraction of valid members (No missing values along time).", False),
        "agree": ("Fraction of valid members agreeing on the sign of change. "
                  + ("Maximum between the positive, negative and no change fractions." if strict_sign
                     else "Maximum between the zero or positive and the zero or negative change fractions."), False),
    }
    parts = {}
    for k, name in enumerate(_lib.ENS_FRACTIONS):
        d, has_test = desc[name]
        attrs = {"description": d, "units": ""}
        if has_test:
            attrs["test"] = str(test)
        parts[name] = _wrap(fut, frac[k].reshape(rest), rest_dims, attrs, name)
    if pvals is not None:
        attrs = {"description": f"P-values from change significance test. {test_str}", "units": ""}
        # apply_ufunc keeps fut's dim order without time
        have = (REALIZATION,) + rest_dims
        pv = pvals.reshape((R,) + rest).permute([have.index(d) for d in p_dims]).contiguous()
        parts["pvals"] = _wrap(fut, pv, p_dims, attrs, "pvals")
    out = _collect(parts, fut)
    if _is_dataset(out):
        out.attrs["description"] = "Significant change and sign of change fractions."
    return out


def robustness_categories(changed_or_fractions, agree=None, valid=None, *, categories=None, ops=None,
                          thresholds=None):
    """Categorical robustness map (ensembles/_robustness.py:336-426): 1-based category of the first matching
    (changed, agree) rule, 99 where none matches or no member is valid.  Elementwise, on the fractions where they
    are (device tensors stay on the device)."""
    if categories is None:
        categories = ["Robust signal", "No change or no signal", "Conflicting signal"]
    if ops is None:
        ops = [(">=", ">="), ("<", None), (">=", "<")]
    if thresholds is None:
        thresholds = [(0.66, 0.8), (0.66, None), (0.66, 0.8)]
    src = changed_or_fractions
    if _is_dataset(src) or isinstance(src, dict):
        changed, agree, valid = src["changed"], src["agree"], src["valid"]
    else:
        changed = src
    cv, av = _raw(changed), _raw(agree)
    torch_like = hasattr(cv, "is_cuda")
    if torch_like:
        import torch
        where = torch.where
        rob = torch.full(cv.shape, 99, dtype=torch.int64, device=cv.device)
    else:
        where = np.where
        rob = np.full(np.shape(cv), 99, dtype=np.int64)
    for i, ((chg_op, agr_op), (chg_thr, agr_thr)) in reversed(list(enumerate(zip(ops, thresholds), 1))):
        if not agr_op:
            cond = _compare(cv, chg_op, chg_thr)
        elif not chg_op:
            cond = _compare(av, agr_op, agr_thr)
        else:
            cond = _compare(cv, chg_op, chg_thr) & _compare(av, agr_op, agr_thr)
        rob = where(cond, i, rob)
    if valid is not None:
        rob = where(_raw(valid) > 0, rob, 99)
    attrs = dict(getattr(changed, "attrs", {}))
    attrs.update(flag_values=list(range(1, len(categories) + 1)), _FillValue=99, flag_descriptions=categories,
                 flag_meanings=" ".join(c.casefold().replace(" ", "_") for c in categories))
    if isinstance(changed, Field) or is_xarray(changed):
        return _wrap(changed, rob, tuple(changed.dims), attrs, getattr(changed, "name", None))
    return rob


def _raw(obj):
    return obj.values if (isinstance(obj, Field) or is_xarray(obj)) else obj


_CMP = {">": "__gt__", "gt": "__gt__", "<": "__lt__", "lt": "__lt__", ">=": "__ge__", "ge": "__ge__",
        "<=": "__le__", "le": "__le__", "==": "__eq__", "eq": "__eq__", "!=": "__ne__", "ne": "__ne__"}


def _compare(a, op, thr):
    if op not in _CMP:
        raise ValueError(f"Operation `{op}` not recognized.")
    return getattr(a, _CMP[op])(thr)
