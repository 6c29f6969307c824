"""Ensemble statistics oracle (ensembles/_base.py, ensembles/_robustness.py) in numpy / scipy.

The reference's ensemble code imports xarray, so it is restated here: the percentiles are
``xclim_oracle.nan_quantile`` along the member axis (the reference's ``calc_perc``) with the sort fixed to IEEE
totalOrder so that the sign of a zero result is defined, the moments a float64
restatement plus xarray's weighted formulas, the robustness fractions a literal float64 restatement of
_robustness.py:218-319 with the t-test p-values from the same float64 statistics through
``scipy.special.stdtr``.  Every sum runs over members (or time steps) in order, as the kernels do.
The member axis is axis 0; robustness series are (R, T, ...).
"""
from __future__ import annotations

import numpy as np
import scipy.special as sps

from . import xclim_oracle as O

QUANTILE_PARAMS = {
    "interpolated_inverted_cdf": (0, 1),
    "hazen": (0.5, 0.5),
    "weibull": (0, 0),
    "linear": (1, 1),
    "median_unbiased": (1 / 3, 1 / 3),
    "normal_unbiased": (3 / 8, 3 / 8),
}


def _total_order_sort(flat):
    """float32 (R, N) sorted along axis 0 in IEEE totalOrder (-0 before +0), NaN last.  np.sort leaves the order
    of -0 and +0 unspecified, and with it the sign of a zero quantile; this fixes it."""
    u = np.ascontiguousarray(flat, dtype=np.float32).view(np.uint32)
    key = np.where(u >> 31 == 1, ~u, u | np.uint32(0x80000000))
    key = np.where(np.isnan(flat), np.uint32(0xFFFFFFFF), key)
    return np.take_along_axis(flat, np.argsort(key, axis=0, kind="stable"), axis=0)


def _nan_quantile_total_order(x, quantiles, alpha, beta):
    """xclim_oracle.nan_quantile (core/utils.py:494-557, R >= 2) with the sort in totalOrder and the maximum of
    :554 the last value in that order: equal to it value for value, and defined to the sign of zero."""
    R = x.shape[0]
    flat = x.reshape(R, -1)
    srt = _total_order_sort(flat)
    n_valid = (R - np.isnan(flat).sum(axis=0)).astype(np.float64)
    cols = np.arange(flat.shape[1])
    vmax = srt[np.maximum(n_valid.astype(np.intp) - 1, 0), cols]
    out = np.empty((len(quantiles), flat.shape[1]), dtype=np.float64)
    with np.errstate(all="ignore"):
        for qi, q in enumerate(quantiles):
            n = np.where(n_valid < 2, np.nan, n_valid)
            vi = n * q + (alpha + q * (1 - alpha - beta)) - 1
            prev = np.floor(vi)
            nxt = prev + 1
            above = vi >= n - 1
            prev, nxt = np.where(above, -1, prev), np.where(above, -1, nxt)
            below = vi < 0
            prev, nxt = np.where(below, 0, prev), np.where(below, 0, nxt)
            isn = np.isnan(vi)
            prev = np.where(isn, -1, prev).astype(np.intp)
            nxt = np.where(isn, -1, nxt).astype(np.intp)
            left, right = srt[prev, cols], srt[nxt, cols]
            gamma = vi - prev
            diff = np.subtract(right, left)
            res = np.where(gamma >= 0.5, np.subtract(right, diff * (1 - gamma)), np.add(left, diff * gamma))
            out[qi] = np.where(np.isnan(res), vmax, res)
    return out.reshape((len(quantiles),) + x.shape[1:])


def percentiles(x, per, alpha=1.0, beta=1.0, min_members=1):
    """(n_per,) + x.shape[1:]: float64 for R >= 2, the input dtype for R == 1 (np.take branch), NaN where fewer
    than min_members members are not NaN (_base.py:329-357)."""
    x = np.asarray(x)
    if x.shape[0] == 1:
        out = np.broadcast_to(x[0], (len(per),) + x.shape[1:]).copy()
    else:
        out = _nan_quantile_total_order(x.astype(np.float32), np.asarray(per, dtype=np.float64) / 100.0, alpha,
                                        beta)
    enough = (~np.isnan(x)).sum(0) >= min_members
    return np.where(enough, out, np.nan).astype(out.dtype)


def _seq_sum(a):
    """sum over axis 0, one member (or step) after the other"""
    s = np.zeros(a.shape[1:], dtype=np.float64)
    for k in range(a.shape[0]):
        s = s + a[k]
    return s


def moments(x, weights=None, min_members=1):
    """(mean, std, min, max) across members (_base.py:178-206): float32 mean / std from float64 sums without
    weights, float64 with xarray's Weighted.mean / .std formulas with them."""
    x = np.asarray(x, dtype=np.float32)
    valid = ~np.isnan(x)
    n = valid.sum(0)
    x64 = x.astype(np.float64)
    with np.errstate(all="ignore"):
        if weights is None:
            sw = n.astype(np.float64)
            m = np.where(n > 0, _seq_sum(np.where(valid, x64, 0.0)) / sw, np.nan)
            d = x64 - m
            sd = np.sqrt(_seq_sum(np.where(valid, d * d, 0.0)) / sw)
            mean, std = m.astype(np.float32), sd.astype(np.float32)
        else:
            w = np.asarray(weights, dtype=np.float64).reshape((-1,) + (1,) * (x.ndim - 1))
            sw = _seq_sum(np.where(valid, w, 0.0))
            sw = np.where(sw != 0.0, sw, np.nan)                       # xarray: _sum_of_weights
            mean = _seq_sum(np.where(valid, x64 * w, 0.0)) / sw
            d = x64 - mean
            std = np.sqrt(_seq_sum(np.where(valid, d * d * w, 0.0)) / sw)
        vmin = np.nanmin(np.where(valid, x, np.inf), axis=0).astype(np.float32)
        vmax = np.nanmax(np.where(valid, x, -np.inf), axis=0).astype(np.float32)
    enough = (n >= min_members) & (n > 0)
    return tuple(np.where(enough, v, np.nan).astype(v.dtype) for v in (mean, std, vmin, vmax))


def _series(a):
    """NaN-omitting float64 (n, mean, ss) along axis 1 of (R, T, ...)"""
    a = np.asarray(a, dtype=np.float32).astype(np.float64)
    valid = ~np.isnan(a)
    n = valid.sum(1)
    with np.errstate(all="ignore"):
        m = np.where(n > 0, _seq_sum(np.moveaxis(np.where(valid, a, 0.0), 1, 0)) / n, np.nan)
        d = a - m[:, None]
        ss = _seq_sum(np.moveaxis(np.where(valid, d * d, 0.0), 1, 0))
    return n, m, ss


def t_pvalue(t, df):
    return 2.0 * sps.stdtr(df, -np.abs(t))


def ttest_1samp_p(n, m, ss, popmean):
    with np.errstate(all="ignore"):
        t = (m - popmean) / np.sqrt(ss / (n - 1) / n)
        return t_pvalue(t, np.where(n >= 2, n - 1, np.nan))


def welch_ttest_p(n1, m1, ss1, n2, m2, ss2):
    with np.errstate(all="ignore"):
        vn1 = ss1 / (n1 - 1) / n1
        vn2 = ss2 / (n2 - 1) / n2
        s = vn1 + vn2
        df = s * s / (vn1 * vn1 / (n1 - 1) + vn2 * vn2 / (n2 - 1))
        df = np.where(np.isnan(df), 1.0, df)
        return t_pvalue((m1 - m2) / np.sqrt(s), df)


def ys_annual_means(ref, poff):
    """(R, P, ...) float32 YS means of (R, T, ...) series: `ref.resample(time="YS").mean()` (NaN-skipping float64
    means rounded once, as the period_reduce kernel)."""
    ref = np.asarray(ref, dtype=np.float32)
    return np.stack([O.resample_reduce(ref[r].astype(np.float64), poff, "mean") for r in range(ref.shape[0])]
                    ).astype(np.float32)


def ipcc_ar6_c_gamma(refy, ys_time):
    """sqrt(2/20) * 1.645 * std of the linearly detrended YS means (_robustness.py:651-654): numpy.polyfit on the
    YS timestamps (xarray's polyfit), the residuals' NaN-skipping std (ddof 0).  refy (R, P, ...) -> (R, ...)."""
    refy = np.asarray(refy, dtype=np.float64)
    x = np.asarray(ys_time, dtype=np.float64)
    flat = np.moveaxis(refy, 1, -1).reshape(-1, x.size)
    sig = np.full(flat.shape[0], np.nan)
    for i, y in enumerate(flat):
        ok = ~np.isnan(y)
        if ok.sum() == 1:
            sig[i] = 0.0
        elif ok.sum() >= 2:
            res = y[ok] - np.polyval(np.polyfit(x[ok], y[ok], 1), x[ok])
            sig[i] = np.sqrt(np.mean(res * res))
    return np.sqrt(2 / 20) * 1.645 * sig.reshape((refy.shape[0],) + refy.shape[2:])


FRACTIONS = ("changed", "positive", "changed_positive", "negative", "changed_negative", "valid", "agree")


def robustness(fut, ref=None, test=None, weights=None, strict_sign=True, changed=None, **kw):
    """_robustness.py:218-319 in float64.  fut / ref: (R, T, ...) series, or fut (R, ...) deltas with ref None.
    Returns (dict of the seven fractions, pvals float64 (R, ...) or None, changed (R, ...)).  ``changed`` may be
    given to evaluate the fractions with another test's flags.  ipcc-ar6-c takes ``poff`` (the YS period offsets
    of ref's time axis) and ``ys_time`` (the YS timestamps), or ``refy`` (the YS means) and ``ys_time``."""
    fut = np.asarray(fut, dtype=np.float32)
    if ref is None:
        delta = fut.astype(np.float64)
        valid = ~np.isnan(delta)
        mr = None
    else:
        nf, mf, ssf = _series(fut)
        nr, mr, ssr = _series(ref)
        delta = mf - mr
        valid = (nf == fut.shape[1]) & (nr == np.asarray(ref).shape[1])
    pvals = None
    with np.errstate(all="ignore"):
        if changed is not None:
            chg = np.asarray(changed, bool)
        elif test is None:
            chg = np.ones(delta.shape, bool)
        elif test == "threshold" and kw.get("abs_thresh") is not None:
            chg = np.abs(delta) > kw["abs_thresh"]
        elif test == "threshold":
            chg = np.abs(delta / mr) > kw["rel_thresh"]
        elif test == "ipcc-ar6-c":
            refy = kw["refy"] if kw.get("refy") is not None else ys_annual_means(ref, kw["poff"])
            chg = np.abs(delta) > ipcc_ar6_c_gamma(refy, kw["ys_time"])
        else:
            if test == "ttest":
                pvals = ttest_1samp_p(nf, mf, ssf, mr)
            elif test == "welch-ttest":
                pvals = welch_ttest_p(nf, mf, ssf, nr, mr, ssr)
            else:
                raise NotImplementedError(test)
            chg = pvals < kw.get("p_change", 0.05)
        R = delta.shape[0]
        w = np.ones(R) if weights is None else np.asarray(weights, dtype=np.float64)
        w = w.reshape((R,) + (1,) * (delta.ndim - 1))
        pos = delta > 0 if strict_sign else delta >= 0
        neg = delta < 0 if strict_sign else delta <= 0

        def wsum(m):
            return _seq_sum(np.where(valid & m, w, 0.0))

        sv = wsum(np.ones(delta.shape, bool))
        pf, nf_ = wsum(pos) / sv, wsum(neg) / sv
        out = {"changed": wsum(chg) / sv, "positive": pf, "changed_positive": wsum(pos & chg) / sv,
               "negative": nf_, "changed_negative": wsum(neg & chg) / sv, "valid": sv / R,
               "agree": np.fmax(np.fmax(pf, nf_), 1 - pf - nf_)}
    return {k: np.nan_to_num(v, nan=0.0, posinf=np.inf, neginf=-np.inf) for k, v in out.items()}, pvals, chg
