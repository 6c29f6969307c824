"""Oracle for the spatial analogues (analog.py): every metric restated in numpy / scipy, in float64.

Each function takes the target sample ``x`` (n, d) and the candidate sample ``y`` (m, d) as ``_metric_overhead``
(:154-170) passes them, returns NaN when either holds a NaN, and raises the reference's ``ValueError`` where the
reference raises.  ``nearest_neighbor`` follows the kernel's stated tie rule (the nearest *other* pooled point,
ties to the lowest pooled index) and its arithmetic: means and stds summed in sample order, the points divided by
sqrt(std_x std_y), squared distances summed in indicator order.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import distance

METRICS = ["seuclidean", "nearest_neighbor", "zech_aslan", "szekely_rizzo", "friedman_rafsky",
           "kolmogorov_smirnov", "kldiv", "mahalanobis"]
MSG_KDTREE = "data must be finite, check for nan or inf values"
MSG_CHKFINITE = "array must not contain infs or NaNs"


def _seq_stats(a):
    """Mean and std(ddof=1) per column, summed in row order (the kernel's col_stats)."""
    s = np.zeros(a.shape[1])
    for row in a:
        s = s + row
    mu = s / a.shape[0]
    q = np.zeros(a.shape[1])
    for row in a:
        e = row - mu
        q = q + e * e
    with np.errstate(all="ignore"):
        return mu, np.sqrt(q / (a.shape[0] - 1))


def target_consts(x, method, VI=None):
    """The per-target constants: var(ddof=1) for seuclidean, the inverse covariance for mahalanobis."""
    x = np.asarray(x, dtype=np.float64)
    with np.errstate(all="ignore"):
        if method == "seuclidean":
            return x.var(axis=0, ddof=1)
        if method == "mahalanobis":
            if VI is not None:
                return np.asarray(VI, dtype=np.float64)
            v = np.cov(x, rowvar=False)        # 0-d for one indicator: np.linalg.inv raises, as in the reference
            try:
                return np.linalg.inv(v)
            except np.linalg.LinAlgError:
                return np.linalg.pinv(v)
    return None


def _pair_dists(a, b, squared=False):
    """Euclidean distances, their squares summed in indicator order."""
    d2 = np.zeros((a.shape[0], b.shape[0]))
    for k in range(a.shape[1]):
        e = a[:, None, k] - b[None, :, k]
        d2 = d2 + e * e
    return d2 if squared else np.sqrt(d2)


def seuclidean(x, y, V=None):
    V = target_consts(x, "seuclidean") if V is None else V
    with np.errstate(all="ignore"):
        t = np.sqrt(1.0 / V) * (x.mean(axis=0) - y.mean(axis=0))
    if not np.isfinite(t).all():
        raise ValueError(MSG_CHKFINITE)
    return float(np.sqrt(np.sum(t * t)))


def nearest_neighbor(x, y):
    _, sx = _seq_stats(x)
    _, sy = _seq_stats(y)
    with np.errstate(all="ignore"):
        s = np.sqrt(sx * sy)
        z = np.vstack([x, y]) / s
    if not np.isfinite(z).all():
        raise ValueError(MSG_KDTREE)
    dist = _pair_dists(z, z, squared=True)
    np.fill_diagonal(dist, np.inf)
    nb = np.argmin(dist, axis=1)          # first of the minima: ties to the lowest pooled index
    n = x.shape[0]
    own = np.arange(z.shape[0]) < n
    return float(np.mean(own == (nb < n)))


def _std_product(x, y):
    with np.errstate(all="ignore"):
        return x.std(axis=0, ddof=1) * y.std(axis=0, ddof=1)


def zech_aslan(x, y, dmin=1e-12):
    n, m = x.shape[0], y.shape[0]
    v = _std_product(x, y)
    with np.errstate(all="ignore"):
        dx = distance.pdist(x, "seuclidean", V=v)
        dy = distance.pdist(y, "seuclidean", V=v)
        dxy = distance.cdist(x, y, "seuclidean", V=v)
        phix = -np.log(dx.clip(dmin)).sum() / (n * (n - 1))
        phiy = -np.log(dy.clip(dmin)).sum() / (m * (m - 1))
        phixy = -np.log(dxy.clip(dmin)).sum() / (n * m)
        return float(phix + phiy - phixy)


def szekely_rizzo(x, y, standardize=True):
    n, m = x.shape[0], y.shape[0]
    with np.errstate(all="ignore"):
        if standardize:
            v = _std_product(x, y)
            sxy = distance.cdist(x, y, "seuclidean", V=v).sum() / (n * m)
            sxx = distance.pdist(x, "seuclidean", V=v).sum() * 2 / n ** 2
            syy = distance.pdist(y, "seuclidean", V=v).sum() * 2 / m ** 2
        else:
            sxy = distance.cdist(x, y).sum() / (n * m)
            sxx = distance.pdist(x).sum() * 2 / n ** 2
            syy = distance.pdist(y).sum() * 2 / m ** 2
        return float(n * m / (n + m) * (sxy + sxy - sxx - syy))


def _ks_pivot(a, b):
    """max over pivots p of a and quadrant codes of |count_a / na - count_b / nb| (the reference's pivot)."""
    w = 2 ** np.arange(a.shape[1])
    ca = ((a[:, None, :] <= a[None, :, :]) * w).sum(-1)     # [pivot, point]
    cb = ((a[:, None, :] <= b[None, :, :]) * w).sum(-1)
    best = 0.0
    for p in range(a.shape[0]):
        codes, inv = np.unique(np.concatenate([ca[p], cb[p]]), return_inverse=True)
        na = np.bincount(inv[:a.shape[0]], minlength=codes.size) * 1.0 / a.shape[0]
        nb = np.bincount(inv[a.shape[0]:], minlength=codes.size) * 1.0 / b.shape[0]
        best = max(best, float(np.max(np.abs(na - nb))))
    return best


def kolmogorov_smirnov(x, y):
    return max(_ks_pivot(x, y), _ks_pivot(y, x))


def _kth(dist, k):
    """k-th (0-based) smallest distance per row, inf where a row has fewer values (cKDTree's fill)."""
    srt = np.sort(dist, axis=1)
    return srt[:, k] if k < srt.shape[1] else np.full(srt.shape[0], np.inf)


def kldiv(x, y, k=1):
    n, d = x.shape
    m = y.shape[0]
    if d > 10:
        raise ValueError(f"Too many dimensions: {d}.")
    if n < 5 or m < 5:
        return np.nan
    if not (np.isfinite(x).all() and np.isfinite(y).all()):
        raise ValueError(MSG_KDTREE)
    r = _kth(_pair_dists(x, x), k)
    s = _kth(_pair_dists(x, y), k - 1)
    with np.errstate(all="ignore"):
        return float(-np.log(r / s).sum() * d / n + np.log(m / (n - 1.0)))


def mahalanobis(x, y, VI=None):
    VI = target_consts(x, "mahalanobis", VI)
    with np.errstate(all="ignore"):
        delta = x.mean(axis=0) - y.mean(axis=0)
        return float(np.sqrt(np.dot(np.dot(delta, VI), delta)))


def metric(method, x, y, **kwargs):
    """`_metric_overhead` (:154-170) then the metric: NaN when either sample holds a NaN."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    if np.isnan(x).any() or np.isnan(y).any():
        return np.nan
    x = np.atleast_2d(x)
    y = np.atleast_2d(y)
    if x.shape[0] == 1:
        x = x.T
    if y.shape[0] == 1:
        y = y.T
    return globals()[method](x, y, **kwargs)
