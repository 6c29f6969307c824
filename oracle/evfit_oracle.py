"""TEST INFRASTRUCTURE: the frequency-analysis fits and transforms restated in numpy / scipy.

* norm: scipy's closed form on the float32 sample, numpy's float32 mean and mean square (bit for bit).
* gumbel_r: the maximum-likelihood scale as the root of scipy's free-loc equation, evaluated in float64 on the
  float64 copy of the sample as scipy does for float64 data (on float32 data scipy evaluates it in float32 and
  its root carries float32 noise),
  found by scipy's own bracket walk and brentq at a tight tolerance; loc from the logsumexp expression.
* genextreme: the optimum of scipy's own ``genextreme.nnlf`` reached by Nelder-Mead from xclim's start (from
  c = 0 where a value lies beyond 1/c), driven to xatol 1e-10.
* transforms: scipy.stats ppf / isf / cdf.

Samples where the likelihood has no maximum (one repeated value, or c >= 1 for genextreme) are NaN.
"""
from __future__ import annotations

import warnings

import numpy as np

PARAM_NAMES = {"norm": ["loc", "scale"], "gumbel_r": ["loc", "scale"], "genextreme": ["c", "loc", "scale"]}


def finite(v):
    v = np.asarray(v, np.float32)
    return v[np.isfinite(v)]


def fit_norm(x):
    m = x.mean(dtype=np.float32)
    return np.array([m, np.sqrt(((x - m) ** 2).mean(dtype=np.float32))], np.float64)


def _gumbel_eq(x32, x64, s):
    lw = -x64 / s
    w = np.exp(lw - lw.max())
    return x64.mean() - np.sum(w * x64) / np.sum(w) - s


def fit_gumbel(x):
    from scipy import optimize, special
    x64 = x.astype(np.float64)
    lb, rb = 0.5, 2.0
    with np.errstate(all="ignore"):
        while np.sign(_gumbel_eq(x, x64, lb)) == np.sign(_gumbel_eq(x, x64, rb)) and (lb > 0 or rb < np.inf):
            lb, rb = lb / 2, rb * 2
        s = optimize.brentq(lambda v: _gumbel_eq(x, x64, v), lb, rb, xtol=1e-300, rtol=4 * np.finfo(float).eps,
                            maxiter=500)
        loc = -s * (special.logsumexp(-x64 / s) - np.log(len(x64)))
    return np.array([loc, s])


def gev_start(x):
    m, v = x.mean(), x.var()
    s = np.sqrt(6 * v) / np.pi
    if not (np.isfinite(s) and s > 0):
        x64 = x.astype(np.float64)
        m, s = x64.mean(), np.sqrt(6 * x64.var()) / np.pi
    return np.array([0.1, float(m - 0.57722 * s), float(s)])


def gev_nnlf(p, x):
    import scipy.stats as st
    return float(st.genextreme.nnlf(p, np.asarray(x, np.float64)))


def fit_gev(x):
    from scipy import optimize
    x64 = x.astype(np.float64)
    p = gev_start(x)
    f = lambda q: gev_nnlf(q, x64)  # noqa: E731
    if not np.isfinite(f(p)):       # a value beyond 1/c: start from the Gumbel law
        p[0] = 0.0
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        r = optimize.minimize(f, p, method="Nelder-Mead", options=dict(xatol=1e-10, fatol=1e-13, maxiter=20000))
        p = r.x
    if not np.isfinite(f(p)) or p[0] >= 1:
        return np.full(3, np.nan)
    return p


def fit(v, dist):
    """One cell: NaN / +-inf dropped, <= 1 value left -> NaN, one repeated value -> NaN (gumbel_r, genextreme)."""
    x = finite(v)
    k = len(PARAM_NAMES[dist])
    if x.size <= 1 or (dist != "norm" and x.min() == x.max()):
        return np.full(k, np.nan)
    p = {"norm": fit_norm, "gumbel_r": fit_gumbel, "genextreme": fit_gev}[dist](x)
    return np.full(k, np.nan) if np.isnan(p).any() else p


def transform(params, dist, kind, q):
    """(nq, C) of scipy's ppf / isf / cdf with the (2 | 3, C) params."""
    import scipy.stats as st
    d = getattr(st, dist)
    q = np.atleast_1d(np.asarray(q, np.float64))[:, None]
    with np.errstate(all="ignore"):
        return getattr(d, kind)(q, *[params[j][None, :] for j in range(params.shape[0])])


def return_levels(params, dist, t=(2, 10, 100)):
    """The mode="max" return levels of fa (isf(1 / t)), (len(t), C)."""
    return transform(params, dist, "isf", 1.0 / np.asarray(t, np.float64))
