"""TEST INFRASTRUCTURE (like everything under oracle/): CPU restatement of detrended quantile mapping (xsdba
``DetrendedQuantileMapping`` with a ``PolyDetrend``, group="time"; PARITY UNPINNED, the same status as EQM and QDM)
and of ``xclim.indices.generic.detrend`` (indices/generic.py:1711-1736).

The trend restates xarray's ``polyfit`` / ``polyval`` on a gap-free daily axis: a Vandermonde matrix of the
nanosecond coordinate, column scaling, ``np.linalg.lstsq`` (``rcond = T * eps`` when the series has no NaN, the
per-column NaN path with numpy's default otherwise), then Horner in the nanosecond coordinate.  Not pinned against
xarray: a cell with an infinite valid value, where this module returns an all-NaN trend.  Train builds on
``xclim_oracle.eqm_train``; the factor of adjust comes from ``scipy.interpolate.interp1d`` itself, called as xsdba's
``_interp_on_quantiles_1D`` calls it (as in qdm_oracle.py).  Used by tests/test_dqm_cpu.py, tests/test_gpu_dqm.py
and bench_extra.py's CPU leg; never by the product path."""
import numpy as np

from .xclim_oracle import eqm_train

NS_PER_DAY = 86400 * 10**9
START_NS = 4018 * NS_PER_DAY      # 1981-01-01, the default start of the daily axis


def _cells(x):
    x = np.asarray(x)
    return x.reshape(x.shape[0], -1)


def _inv(m, kind):
    """xsdba.utils.invert: -m ("+") or 1 / m ("*") in float32."""
    m = np.asarray(m, dtype=np.float32)
    with np.errstate(all="ignore"):
        return -m if kind == "+" else (np.float32(1) / m).astype(np.float32)


def _apply(x, c, kind):
    """xsdba.utils.apply_correction in float32: x + c or x * c."""
    with np.errstate(all="ignore"):
        return (x + c if kind == "+" else x * c).astype(np.float32)


def cell_mean(x):
    """NaN-skipping mean of every cell as float32: the float64 sum of the valid values, taken in time order, over
    their count, rounded once (what xc_period_reduce_f32 computes for one period with the mean statistic)."""
    x2 = _cells(x).astype(np.float64)
    ok = ~np.isnan(x2)
    s = np.cumsum(np.where(ok, x2, 0.0), axis=0)[-1]
    n = ok.sum(axis=0)
    with np.errstate(all="ignore"):
        return np.where(n > 0, s / np.maximum(n, 1), np.nan).astype(np.float32).reshape(np.asarray(x).shape[1:])


def dqm_train(ref, hist, nquantiles=20, kind="+"):
    """DetrendedQuantileMapping.train(group="time"): EQM's quantiles of ``refn = float32(ref (+|*) inv(m_ref))``
    and ``histn`` (likewise), ``scaling = m_ref - m_hist`` ("+") or ``m_ref / m_hist`` ("*").
    Returns ``(af, hist_q, scaling)``."""
    ref, hist = np.asarray(ref, np.float32), np.asarray(hist, np.float32)
    m_ref, m_hist = cell_mean(ref), cell_mean(hist)
    refn, histn = _apply(ref, _inv(m_ref, kind), kind), _apply(hist, _inv(m_hist, kind), kind)
    af, hist_q = eqm_train(refn, histn, nquantiles, kind)
    with np.errstate(all="ignore"):
        scaling = (m_ref - m_hist if kind == "+" else m_ref / m_hist).astype(np.float32)
    return af, hist_q, scaling


def poly_trend(y, degree, start_ns=START_NS):
    """xarray ``polyval(time, y.polyfit("time", degree))`` for a daily axis starting ``start_ns`` nanoseconds after
    1970-01-01 (1981-01-01 by default), float64 (T, ...).  All NaN for a cell without valid values or with an infinite one."""
    y2 = _cells(y).astype(np.float64)
    T, C = y2.shape
    x = start_ns + np.arange(T, dtype=np.float64) * NS_PER_DAY
    lhs = np.vander(x, degree + 1)
    scale = np.sqrt((lhs * lhs).sum(axis=0))
    lhs = lhs / scale
    coef = np.full((degree + 1, C), np.nan)
    for c in range(C):
        col = y2[:, c]
        nan = np.isnan(col)
        if nan.all() or np.isinf(col[~nan]).any():
            continue
        if nan.any():
            sol = np.linalg.lstsq(lhs[~nan], col[~nan], rcond=None)[0]
        else:
            sol = np.linalg.lstsq(lhs, col, rcond=T * np.finfo(np.float64).eps)[0]
        coef[:, c] = sol / scale
    res = np.zeros((T, C)) + coef[0]
    for k in range(1, degree + 1):
        res = res * x[:, None] + coef[k]
    return res.reshape(np.asarray(y).shape)


def basis_u(T):
    """The fit basis of the kernels: u_t = (2t - (T - 1)) / max(T - 1, 1), float64."""
    return (2 * np.arange(T) - (T - 1)) / float(max(T - 1, 1))


def trend_from_coef(coef, T):
    """The trend (T, C) from the kernel's coefficients (D + 1, C), row k = coefficient of u^k: Horner from the
    highest row, ``((c2 u + c1) u + c0)``, one float64 operation at a time."""
    coef = np.asarray(coef, dtype=np.float64)
    u = basis_u(T)[:, None]
    res = np.zeros((T, coef.shape[1])) + coef[-1]
    for k in range(coef.shape[0] - 2, -1, -1):
        res = res * u + coef[k]
    return res


def dqm_adjust(sim, af, hist_q, scaling, kind="+", interp="nearest", detrend=1, coef=None, start_ns=START_NS):
    """DetrendedQuantileMapping.adjust(extrapolation="constant", detrend=<degree>) per cell:
    ``y = float32(sim (+|*) scaling)``; ``tau`` = poly_trend(y, detrend), or trend_from_coef(coef) when the kernel's
    coefficients are given; ``d = y - tau`` or ``y * (1 / tau)`` in float64; ``f = interp1d(hist_q[ok], af[ok],
    kind=interp, bounds_error=False, fill_value=(first, last))(d)`` as float32, ``ok`` excluding NaN in either
    table; ``scen = float32((d (+|*) f) (+|*) tau)``.  Returns float32 scen shaped like sim."""
    from scipy.interpolate import interp1d
    sim = np.asarray(sim, dtype=np.float32)
    s2 = _cells(sim)
    T, C = s2.shape
    af2 = np.asarray(af, np.float32).reshape(np.asarray(af).shape[0], -1)
    hq2 = np.asarray(hist_q, np.float32).reshape(af2.shape[0], -1)
    y = _apply(s2, np.asarray(scaling, np.float32).reshape(-1), kind)
    tau = trend_from_coef(coef, T) if coef is not None else poly_trend(y, detrend, start_ns)
    with np.errstate(all="ignore"):
        d = y - tau if kind == "+" else y * (1.0 / tau)
        fac = np.full((T, C), np.nan, dtype=np.float32)
        for c in range(C):
            ok = ~(np.isnan(hq2[:, c]) | np.isnan(af2[:, c]))
            m = ~np.isnan(d[:, c])
            if not ok.any() or not m.any():
                continue
            yv = af2[ok, c]
            f = interp1d(hq2[ok, c], yv, kind=interp, bounds_error=False, fill_value=(yv[0], yv[-1]))
            fac[m, c] = f(d[m, c])
        f64 = fac.astype(np.float64)
        scen = (d + f64) + tau if kind == "+" else (d * f64) * tau
    return scen.astype(np.float32).reshape(sim.shape)


def detrend(x, degree=1, start_ns=START_NS):
    """generic.detrend(x, "time", degree): ``x - trend`` in float64 (float32 data minus the float64 trend)."""
    x = np.asarray(x, dtype=np.float32)
    return x.astype(np.float64) - poly_trend(x, degree, start_ns)
