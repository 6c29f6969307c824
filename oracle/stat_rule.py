"""The per-period float statistic rule of the streaming kernels, restated in numpy float64.  TEST INFRASTRUCTURE.

Every kernel that reduces a period to a float statistic (``period_reduce_kernel``, ``StatAcc`` in the rolling and
daily-range kernels, ``RunAcc`` in the run-length kernels, ``period_run_maxsum_kernel`` and the R95pTOT sums of
``period_count_thr_kernel``) promises the same arithmetic in its comments:

  * values are float32; NaN values are skipped;
  * the sum and the sum of squares are float64, added one value at a time in time order (``np.sum`` pairs the
    values up and must not stand in for them; ``v * v`` of a float32 ``v`` is exact in float64);
  * each result is rounded to float32 once:  sum ``f32(s)``, mean ``f32(s / n)``, count ``n``;
  * ``var = q / n - mean * mean`` with every operation rounded (no fused multiply-add), clamped at 0 (a NaN
    difference, from infinite values, is 0 too), ``std = f32(sqrt(var))``;
  * mean, min, max, std and var of no values are NaN; the sum of none is 0.

The functions below loop over time and are vectorised across cells, so that every sum is sequential.
``tests/test_stat_rule.py`` checks them against the reference restatements of ``xclim_oracle`` and
``etccdi_oracle``; ``tests/test_gpu_stat_rule.py`` holds the kernels to them bit for bit.
"""
from __future__ import annotations

import numpy as np

from oracle import xclim_oracle as O

F32 = np.float32
STATS = ("sum", "mean", "min", "max", "std", "var", "count")


def _f32(a):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(a, dtype=np.float64).astype(np.float32)


def var_of(n, s, q):
    """``max(0, fl(q / n) - fl(mean * mean))`` in float64 with ``mean = fl(s / n)`` (NaN where n == 0): numpy never
    fuses the multiply with the subtraction.  A NaN difference is clamped to 0, as the kernels' select does."""
    n = np.asarray(n, dtype=np.float64)
    with np.errstate(all="ignore"):
        mean = np.asarray(s, dtype=np.float64) / n
        var = np.asarray(q, dtype=np.float64) / n - mean * mean
        var = np.where(var > 0.0, var, 0.0)
    return np.where(n > 0, var, np.nan)


def transform(x, kind="none", op=">", thr=0.0):
    """The fused transforms of ``period_reduce_kernel``, in float32: ``excess`` is ``(x - t).clip(0)`` for > / >=
    and ``(t - x).clip(0)`` for < / <= with NaN kept; ``where`` keeps x where ``x op t`` and is NaN elsewhere."""
    x = np.asarray(x, dtype=np.float32)
    if kind == "none":
        return x
    t = F32(thr)
    with np.errstate(all="ignore"):
        if kind == "excess":
            d = (x - t) if op in (">", ">=") else (t - x)
            return np.where(np.isnan(d), d, np.maximum(d, F32(0))).astype(np.float32)
        if kind == "where":
            return np.where(O.compare(x, op, t), x, F32(np.nan)).astype(np.float32)
    raise ValueError(f"unknown transform {kind!r}")


def _moments(blk):
    """n, sequential float64 s and q, float32 min and max of the non-NaN values of blk (time on axis 0)."""
    shape = blk.shape[1:]
    n = np.zeros(shape, np.int64)
    s = np.zeros(shape, np.float64)
    q = np.zeros(shape, np.float64)
    mn = np.full(shape, np.inf, np.float32)
    mx = np.full(shape, -np.inf, np.float32)
    with np.errstate(all="ignore"):
        for v in blk:
            ok = ~np.isnan(v)
            v64 = v.astype(np.float64)
            n += ok
            s = s + np.where(ok, v64, 0.0)
            q = q + np.where(ok, v64 * v64, 0.0)
            mn = np.fmin(mn, v)
            mx = np.fmax(mx, v)
    return n, s, q, mn, mx


def period_stat(x, poff, stat, kind="none", op=">", thr=0.0):
    """The statistic ``stat`` of every period ``[poff[p], poff[p+1])`` (an empty period included) of the float32
    values ``x`` after the transform ``kind``: float32 ``(P, ...)``."""
    v = transform(x, kind, op, thr)
    out = []
    for s0, e0 in O._groups(poff):
        n, s, q, mn, mx = _moments(v[s0:e0])
        with np.errstate(all="ignore"):
            if stat == "sum":
                r = _f32(s)
            elif stat == "count":
                r = n.astype(np.float32)
            elif stat == "mean":
                r = np.where(n > 0, _f32(s / np.maximum(n, 1)), F32(np.nan))
            elif stat in ("min", "max"):
                r = np.where(n > 0, mn if stat == "min" else mx, F32(np.nan))
            elif stat == "var":
                r = _f32(var_of(n, s, q))
            elif stat == "std":
                r = _f32(np.sqrt(var_of(n, s, q)))
            else:
                raise ValueError(f"unknown statistic {stat!r}")
        out.append(np.asarray(r, dtype=np.float32))
    return np.stack(out, axis=0)


def range_stat(lo, hi, poff, stat, variability=False):
    """``period_range_stat_kernel``: the statistic of ``d = hi - lo`` (float32), or with ``variability`` of
    ``|d[t] - d[t-1]|`` (float32; a period's first difference reaches into the previous period, the series' first
    step has none)."""
    with np.errstate(all="ignore"):
        d = np.asarray(hi, dtype=np.float32) - np.asarray(lo, dtype=np.float32)
        if variability:
            prev = np.concatenate([np.full((1,) + d.shape[1:], np.nan, np.float32), d[:-1]])
            d = np.abs(d - prev)
    return period_stat(d, poff, stat)


def run_mean(n, s):
    """``run_mean`` of runstat.cuh: n runs of total length s, 0 when there is none."""
    n = np.asarray(n, dtype=np.float64)
    with np.errstate(all="ignore"):
        return np.where(n > 0, _f32(np.asarray(s, np.float64) / n), F32(0))


def run_std(n, s, q):
    """``run_std`` of runstat.cuh: n runs, total length s, sum of squared lengths q; 0 when there is none."""
    with np.errstate(invalid="ignore"):
        return np.where(np.asarray(n) > 0, _f32(np.sqrt(var_of(n, s, q))), F32(0))


def run_stat(da, reducer, window, poff=None, index="first"):
    """The ``mean`` / ``std`` reducers of the run lengths >= window, drop-in for ``O.rle_statistics`` (so that
    ``O.resample_and_rl`` applies the period rules): the run lengths are ``O.rle``'s, the integer sums exact."""
    d = O.rle(da, index=index)
    groups = [(0, d.shape[0])] if poff is None else O._groups(poff)
    out = []
    for s0, e0 in groups:
        blk = d[s0:e0]
        with np.errstate(invalid="ignore"):
            take = blk >= window
        L = np.where(take, blk, 0).astype(np.int64)
        n, s, q = take.sum(axis=0), L.sum(axis=0), (L * L).sum(axis=0)
        out.append(run_mean(n, s) if reducer == "mean" else run_std(n, s, q))
    return out[0] if poff is None else np.stack(out, axis=0)


def run_maxsum(x, poff, op, thr, window, resample_before_rl=True):
    """``period_run_maxsum_kernel``: the largest float64 sum, in time order, of the float32 excess
    ``(x - t).clip(0)`` (> / >=) or ``(t - x).clip(0)`` (< / <=) over a run of positive excess at least ``window``
    steps long, rounded to float32 once; 0 when there is none.  With ``resample_before_rl`` the runs are cut at the
    period edges, else a run belongs to the period of its first step and keeps its full length."""
    e = transform(x, "excess", op, thr)
    e = np.where(np.isnan(e), F32(0), e)
    T, C = e.shape
    poff = np.asarray(poff)
    P = len(poff) - 1
    period_of = np.full(T, -1, np.int64)
    for p in range(P):
        period_of[poff[p]:poff[p + 1]] = p
    starts = set(int(t) for t in poff)
    best = np.zeros((P, C), np.float64)
    cur = np.zeros(C, np.int64)
    rs = np.zeros(C, np.float64)
    first = np.zeros(C, np.int64)

    def close(sel):
        # the run of each selected cell ends: it counts for the period of its first step (none before poff[0])
        p = period_of[first]
        c = np.nonzero(sel & (cur >= window) & (p >= 0))[0]
        best[p[c], c] = np.fmax(best[p[c], c], rs[c])

    with np.errstate(over="ignore"):
        for t in range(T):
            if resample_before_rl and t in starts:
                close(cur > 0)
                cur[...] = 0
                rs[...] = 0.0
            inrun = e[t] > 0
            close(~inrun & (cur > 0))
            first = np.where(inrun & (cur == 0), t, first)
            rs = np.where(inrun, rs + e[t].astype(np.float64), 0.0)
            cur = np.where(inrun, cur + 1, 0)
        close(cur > 0)
    return _f32(best)


def sums_thr(x, poff, op, thr_rows, wet):
    """The two R95pTOT sums of ``period_count_thr_kernel<..., SUMS>``: per period the float64 sums, in time order,
    of the x with ``float64(x) op thr_rows`` (a float64 threshold per step and cell: a day-of-year table already
    indexed by the steps' day of year, or one row per cell broadcast) and of the x with ``x op float32(wet)``, each
    rounded to float32 once."""
    x = np.asarray(x, dtype=np.float32)
    thr_rows = np.broadcast_to(np.asarray(thr_rows, dtype=np.float64), x.shape)
    w = F32(wet)
    s_thr, s_wet = [], []
    for s0, e0 in O._groups(poff):
        a = np.zeros(x.shape[1:], np.float64)
        b = np.zeros(x.shape[1:], np.float64)
        with np.errstate(all="ignore"):
            for t in range(s0, e0):
                v = x[t].astype(np.float64)
                a = a + np.where(O.compare(v, op, thr_rows[t]), v, 0.0)
                b = b + np.where(O.compare(x[t], op, w), v, 0.0)
        s_thr.append(_f32(a))
        s_wet.append(_f32(b))
    return np.stack(s_thr, axis=0), np.stack(s_wet, axis=0)
