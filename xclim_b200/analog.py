"""Spatial analogues behind the signature of ``xclim.analog.spatial_analogs`` (analog.py).

The dissimilarity between the target sample(s) and the candidate sample of every grid cell runs as one CUDA
kernel (include/xclim_b200.h a1): a CTA holds 32 adjacent cells' samples in shared memory and a warp reduces one
cell.  ``target`` and ``candidates`` are xr.Datasets, or dicts of Fields / DataArrays standing in for one; their
variables are the indicators, stacked in variable order.  The samples lie along ``dist_dim`` (any position, any
length on either side).  Host-backed candidates are staged to the device whole.  The per-target constants of
``seuclidean`` (the variance) and ``mahalanobis`` (the inverse covariance) are computed on the host in float64.
"""
from __future__ import annotations

import numpy as np

from . import _lib, device
from .ensembles import _is_dataset, _variables
from .field import Field, is_xarray
from . import field as _field
from .options import OPTIONS

#: the reference's metric names, in its order (analog.py registers them in this order)
metrics = ["seuclidean", "nearest_neighbor", "zech_aslan", "szekely_rizzo", "friedman_rafsky",
           "kolmogorov_smirnov", "kldiv", "mahalanobis"]

#: keyword arguments of each metric and their defaults (analog.py :181-628)
_KWARGS = {"seuclidean": {}, "nearest_neighbor": {}, "zech_aslan": {"dmin": 1e-12},
           "szekely_rizzo": {"standardize": True}, "kolmogorov_smirnov": {}, "kldiv": {"k": 1},
           "mahalanobis": {"VI": None}}

_UNSUPPORTED = {
    "friedman_rafsky": "friedman_rafsky needs scikit-learn's kneighbors_graph, and its minimum spanning tree is not "
                       "unique under ties, so neither is its count of cross-sample edges: not supported",
}

#: device on which host candidates are staged (the CPU tests substitute their stand-ins)
_DEVICE = "cuda"

MSG_KDTREE = "data must be finite, check for nan or inf values"
MSG_CHKFINITE = "array must not contain infs or NaNs"


def _host(values):
    if hasattr(values, "detach"):
        return values.detach().cpu().numpy()
    return np.asarray(values)


def _stack(variables: dict, dist_dim: str, role: str):
    """The variables' values with dist_dim moved last and the indicators stacked after it: (rest..., n, d) as a
    numpy array or a torch tensor, with the rest dims."""
    dims = None
    parts = []
    for name, da in variables.items():
        d = tuple(da.dims)
        if dist_dim not in d:
            raise ValueError(f"the {role} variable `{name}` has no `{dist_dim}` dimension: {d}")
        if dims is None:
            dims = d
        elif d != dims:
            raise ValueError(f"the {role} variables must share their dims: {dims} and {d}")
        parts.append(da.values)
    ax = dims.index(dist_dim)
    rest = tuple(x for x in dims if x != dist_dim)
    if all(hasattr(v, "is_cuda") for v in parts):
        import torch
        return torch.stack([v.movedim(ax, -1) for v in parts], dim=-1), rest
    return np.stack([np.moveaxis(_host(v), ax, -1) for v in parts], axis=-1), rest


def _params(method, kwargs):
    allowed = _KWARGS[method]
    for k in kwargs:
        if k not in allowed:
            raise TypeError(f"{method}() got an unexpected keyword argument '{k}'")
    kw = {**allowed, **kwargs}
    if method == "zech_aslan":
        return float(kw["dmin"]), kw
    if method == "szekely_rizzo":
        return float(bool(kw["standardize"])), kw
    if method == "kldiv":
        k = kw["k"]
        if np.iterable(k):
            raise NotImplementedError("kldiv with a sequence of k returns one value per k, which the reference's "
                                      "apply_ufunc with a scalar output cannot take either: not supported")
        if int(k) != k or k < 1:
            raise ValueError(f"kldiv needs a positive integer k, got {k}")
        if k > _lib.AN_KLDIV_MAX_K:
            raise NotImplementedError(f"kldiv keeps at most {_lib.AN_KLDIV_MAX_K} neighbours per point: k = {k} "
                                      "is not supported")
        return float(k), kw
    return 0.0, kw


def _target_consts(tk, method, VI):
    """(K, d) variances (seuclidean) or (K, d, d) inverse covariances (mahalanobis) of the float64 targets, as
    analog.py :213 and :620-627 compute them per call; None for the other methods."""
    K, n, d = tk.shape
    if method == "seuclidean":
        with np.errstate(all="ignore"):
            return tk.var(axis=1, ddof=1)
    if method != "mahalanobis":
        return None
    if VI is not None:
        if not isinstance(VI, np.ndarray):
            raise AttributeError("VI not a matrix")
        return np.broadcast_to(np.asarray(VI, dtype=np.float64), (K, d, d)).copy()
    out = np.full((K, d, d), np.nan)
    for t in range(K):
        if np.isnan(tk[t]).any():       # the pair is NaN before the covariance is taken (:154-156)
            continue
        with np.errstate(all="ignore"):
            v = np.cov(tk[t], rowvar=False)
            try:
                out[t] = np.linalg.inv(v)
            except np.linalg.LinAlgError:
                if v.ndim < 2:          # one indicator: np.linalg.inv raises on the 0-d covariance, as in the reference
                    raise
                out[t] = np.linalg.pinv(v)
    return out


def spatial_analogs(target, candidates, dist_dim="time", method="kldiv", **kwargs):
    """Dissimilarity between the target sample(s) and the candidate sample of every cell (analog.py:21-105).

    Output dims: the target's dims other than ``dist_dim`` (one plane per target site), then the candidates';
    float64, named ``dissimilarity``.  Where the reference raises for one cell, the whole call raises."""
    if not isinstance(dist_dim, str):
        raise NotImplementedError("dist_dim must be one dimension name: stacking several dims into a multi-index "
                                  "is not supported (pass a pre-stacked single dim)")
    tvars, cvars = _variables(target), _variables(candidates)
    if list(tvars) != list(cvars):
        raise ValueError(f"cannot align objects with join='exact' where index/labels/sizes are not equal along "
                         f"these coordinates (dimensions): '_indices' ('_indices',): target {list(tvars)}, "
                         f"candidates {list(cvars)}")
    if method not in metrics:
        raise ValueError(f"Method `{method}` is not implemented. Available methods are: {','.join(metrics)}.")
    if method in _UNSUPPORTED:
        raise NotImplementedError(_UNSUPPORTED[method])
    param, kw = _params(method, kwargs)

    tv, t_rest = _stack(tvars, dist_dim, "target")
    cv, c_rest = _stack(cvars, dist_dim, "candidates")
    n, d = int(tv.shape[-2]), int(tv.shape[-1])
    m = int(cv.shape[-2])
    if int(cv.shape[-1]) != d:
        raise AttributeError("Shape mismatch")
    if method == "kldiv" and d > 10:
        raise ValueError(f"Too many dimensions: {d}.")
    t_shape, c_shape = tuple(tv.shape[:-2]), tuple(cv.shape[:-2])
    K, C = int(np.prod(t_shape, dtype=np.int64)), int(np.prod(c_shape, dtype=np.int64))

    import torch
    tk = np.ascontiguousarray(_host(tv).reshape(K, n, d), dtype=np.float32)
    consts = _target_consts(tk.astype(np.float64), method, kw.get("VI"))
    dev = cv.device if hasattr(cv, "is_cuda") and cv.is_cuda else _DEVICE
    if hasattr(cv, "is_cuda"):
        y = cv.to(torch.float32).reshape(C, m, d).permute(1, 2, 0).contiguous().to(dev)
    else:
        y = torch.from_numpy(np.ascontiguousarray(np.moveaxis(_host(cv).reshape(C, m, d), 0, -1),
                                                  dtype=np.float32)).to(dev)
    cst = None if consts is None else torch.from_numpy(np.ascontiguousarray(consts.reshape(K, -1))).to(dev)
    out, status = device.analog(torch.from_numpy(tk).to(dev), y, _lib.AN_METHODS[method], param, cst)
    if status & _lib.AN_STATUS_NOT_FINITE:
        raise ValueError(MSG_KDTREE)
    if status & _lib.AN_STATUS_CHKFINITE:
        raise ValueError(MSG_CHKFINITE)

    dims = t_rest + c_rest
    vals = out.reshape(t_shape + c_shape)
    template = next(iter(cvars.values()))
    xr_out = is_xarray(template) or _is_dataset(candidates)
    if not (OPTIONS["device_outputs"] and not xr_out):
        vals = vals.cpu().numpy()
    attrs = {"long_name": f"Dissimilarity between target and candidates, using metric {method}.",
             "indices": ",".join(str(v) for v in tvars), "metric": method}
    coords = {}
    for src, rest in ((next(iter(tvars.values())), t_rest), (template, c_rest)):
        for dim in rest:
            if dim in getattr(src, "coords", {}):
                coords[dim] = src.coords[dim]
    if xr_out:
        return _field.xr.DataArray(vals, dims=dims, coords=coords, attrs=attrs, name="dissimilarity")
    return Field(vals, dims, None, coords, attrs, "dissimilarity")
