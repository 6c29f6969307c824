"""Standardized indices (SPI / SPEI) restated in numpy / scipy -- indices/stats.py:770-1197.

* ``fit_sample``: one (cell, group) sample through ``_fitfunc_1d`` (:45-112) and ``_fit_start`` (:576-684) for
  gamma / fisk / lognorm with method APP, and scipy's ``gamma_gen.fit`` / ``lognorm_gen.fit`` for method ML with
  a fixed ``floc`` (no optimiser runs there: a ``brentq`` root for gamma, closed forms for lognorm).
* ``numpy_logs``: True evaluates every float32 log / exp with numpy (the reference's own arithmetic); False
  rounds the float64 function once to float32, the rule the kernels follow (numpy's float32 log / exp are SIMD
  code that differs between CPUs).  The same switch picks ``m**3`` (numpy's float32 power) or the float64
  product rounded once for the fisk moments.
* ``rolling_mean``: ``rolling(time=window).mean(skipna=False)`` (:831-832) with the kernels' convention, a float64
  window sum divided by the window and rounded to float32.
* ``fit_groups`` / ``transform``: the groupby of :944-953 on a (T, C) series with an integer group per step
  (-1 = masked by the indexer), and :1155-1191 through ``scipy.stats.<dist>.cdf`` and ``scipy.special.ndtri``.
"""
from __future__ import annotations

import warnings

import numpy as np

CLIP = 8.21


class FitDataError(ValueError):
    """scipy.stats FitDataError (a ValueError): a value outside the support of the fixed-loc distribution."""


def _log(x, numpy_logs):
    if numpy_logs:
        return np.log(x)
    return np.asarray(np.log(np.asarray(x, np.float64)), np.float32)[()]


def _exp(x, numpy_logs):
    if numpy_logs:
        return np.exp(x)
    return np.asarray(np.exp(np.asarray(x, np.float64)), np.float32)[()]


def _cube(m, numpy_logs):
    if numpy_logs:
        return m ** 3
    m64 = np.float64(m)
    return np.float32(m64 * m64 * m64)


def _square(m, numpy_logs):
    return m ** 2 if numpy_logs else m * m


def gamma_ml_bracket(s, numpy_logs=False):
    """scipy gamma_gen.fit: the float32 estimate of the shape and its +-40 % bracket."""
    with np.errstate(all="ignore"):
        aest = (3 - s + np.sqrt(_square(s - 3, numpy_logs) + 24 * s)) / (12 * s)
        return aest, aest * (1 - 0.4), aest * (1 + 0.4)


def gamma_ml_root(s, xa, xb):
    """The brentq call of gamma_gen.fit (defaults xtol 2e-12, rtol 4 eps)."""
    import scipy.special as sc
    from scipy import optimize
    return optimize.brentq(lambda a: np.log(a) - sc.digamma(a) - s, xa, xb, disp=0)


def fit_sample(arr, dist, method, floc, numpy_logs=True):
    """(shape, loc, scale) float64 of one float32 sample (NaN already standing for the dropped zeros when
    zero-inflated).  Raises FitDataError / ValueError / NotImplementedError where the reference raises or
    hands the sample to scipy's generic optimiser."""
    x = np.ma.masked_invalid(np.asarray(arr, np.float32)).compressed()
    if len(x) <= 1:
        return np.full(3, np.nan)
    with np.errstate(all="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if method == "APP":
            x_pos = x - floc
            x_pos = x_pos[x_pos > 0]
            if dist == "gamma":
                m = x_pos.mean()
                A = _log(m, numpy_logs) - _log(x_pos, numpy_logs).mean()
                a0 = (1 + np.sqrt(1 + 4 * A / 3)) / (4 * A)
                params = [a0, floc, m / a0]
            elif dist == "fisk":
                m = x_pos.mean()
                m2 = (x_pos ** 2).mean()
                scale0 = 2 * _cube(m, numpy_logs) / (m2 + _square(m, numpy_logs))
                c0 = np.pi * m / np.sqrt(3) / np.sqrt(m2 - _square(m, numpy_logs))
                params = [c0, floc, scale0]
            else:
                lx = _log(x_pos, numpy_logs)
                params = [lx.std(), floc, _exp(lx.mean(), numpy_logs)]
        elif dist == "gamma":
            if np.any(x <= floc):
                raise FitDataError("Invalid values in `data`.  Maximum likelihood estimation with 'gamma' requires "
                                   f"that {floc!r} < (x - loc)/scale  < inf for each x in `data`.")
            data = x - floc if floc != 0 else x
            xbar = data.mean()
            s = _log(xbar, numpy_logs) - _log(data, numpy_logs).mean()
            _, xa, xb = gamma_ml_bracket(s, numpy_logs)
            a = gamma_ml_root(s, xa, xb)
            params = [a, floc, xbar / a]
        elif dist == "lognorm":
            if floc >= x.min():
                raise FitDataError("Invalid values in `data`.  Maximum likelihood estimation with 'lognorm' requires "
                                   "that 0.0 < (x - loc)/scale  < inf for each x in `data`.")
            ln = _log(x - floc, numpy_logs)
            scale = _exp(ln.mean(), numpy_logs)
            shape = np.sqrt(np.mean((ln - _log(scale, numpy_logs)) ** 2))
            if not (shape > 0 and scale > 0):
                raise NotImplementedError("lognorm ML with a fixed loc on a sample of zero spread: scipy falls "
                                          "back to its generic optimiser")
            params = [shape, floc, scale]
        else:
            raise NotImplementedError(f"{dist} {method}")
    params = np.asarray(params, dtype=np.float64)
    if np.isnan(params).any():
        params[:] = np.nan
    return params


def rolling_mean(x, window):
    """(T, C) float32 -> rolled float32 series: NaN for t < window - 1 or any NaN in the window."""
    x = np.asarray(x, np.float32)
    if window <= 1:
        return x.copy()
    T = x.shape[0]
    out = np.full(x.shape, np.nan, np.float32)
    x64 = x.astype(np.float64)
    with np.errstate(all="ignore"):
        for t in range(window - 1, T):
            out[t] = (x64[t - window + 1:t + 1].sum(axis=0) / window).astype(np.float32)
    return out


def fit_groups(y, group_of_step, G, cal, dist, method, zero_inflated, floc, numpy_logs=False):
    """Params (G, 3, C), n_zeros / n_notnull (G, C) int64 of the (T, C) float32 series ``y`` over the steps in
    ``cal`` (a slice) whose group is >= 0 (stats.py:944-953)."""
    y = np.asarray(y, np.float32)
    T, C = y.shape
    g = np.asarray(group_of_step)[cal]
    yc = y[cal]
    params = np.full((G, 3, C), np.nan)
    nz = np.zeros((G, C), np.int64)
    nn = np.zeros((G, C), np.int64)
    for k in range(G):
        blk = yc[g == k]
        nz[k] = (blk == 0).sum(axis=0)
        nn[k] = (~np.isnan(blk)).sum(axis=0)
        if zero_inflated:
            blk = np.where(blk != 0, blk, np.float32(np.nan))
        for c in range(C):
            params[k, :, c] = fit_sample(blk[:, c], dist, method, floc, numpy_logs)
    return params, nz, nn


def transform(y, group_of_step, params, dist, n_zeros=None, n_notnull=None, interp=1.0, alpha=0.0, beta=1.0):
    """(T, C) float64 standardized index (stats.py:1155-1191) through scipy."""
    import scipy.stats as st
    y = np.asarray(y, np.float32)
    gos = np.asarray(group_of_step)
    ok = gos >= 0
    gi = np.where(ok, gos, 0)
    shape, loc, scale = (params[gi][:, j, :] for j in range(3))
    shape, loc, scale = (np.where(ok[:, None], v, np.nan) for v in (shape, loc, scale))
    dfun = getattr(st, dist)
    with np.errstate(all="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if n_zeros is not None:
            mask = y != 0
            prob_nonzero = dfun.cdf(np.where(mask, y, np.float32(np.nan)), shape, loc, scale)
            nz = np.asarray(n_zeros)[gi]
            nn = np.asarray(n_notnull)[gi]
            den = nn + 1 - alpha - beta
            r1 = (1 - alpha) / den
            rn = (nz - alpha) / den
            rf = (1 - interp) * r1 + interp * rn
            probs = np.where(mask, rn + ((1 - rn) * prob_nonzero), rf)
            probs = np.where(ok[:, None], probs, np.nan)
        else:
            probs = dfun.cdf(y, shape, loc, scale)
        out = st.norm.ppf(probs)
    return np.clip(out, -CLIP, CLIP)
