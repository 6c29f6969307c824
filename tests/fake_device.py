"""TEST INFRASTRUCTURE: a CPU stand-in for ``xclim_b200.device`` built on the oracle.

``install(monkeypatch)`` replaces the device-layer functions by numpy/oracle equivalents working
on CPU torch tensors, so that the HOST layer (units, thresholds, operators, period offsets,
wrapping, attrs, dtypes, option handling) can be exercised by the ``-m "not gpu"`` suite.  It proves
nothing about the kernels -- those are checked by the ``-m gpu`` tests through the C ABI -- and
nothing outside ``tests/`` may import it.
"""
import numpy as np
import torch

from oracle import xclim_oracle as O
from xclim_b200 import _lib

OP_NAME = {0: ">", 1: "<", 2: ">=", 3: "<=", 4: "==", 5: "!="}
RED_NAME = {v: k for k, v in _lib.RL_REDUCERS.items()}
STAT_NAME = {0: "sum", 1: "mean", 2: "min", 3: "max", 4: "std", 5: "var", 6: "count"}


def _np(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def _cond(x, op_code, thr, cmp_f64=False):
    if op_code == _lib.OP_ISNAN:
        return np.isnan(x)
    if op_code == _lib.OP_NOTNAN:
        return ~np.isnan(x)
    return O.compare(x, OP_NAME[op_code], np.float64(thr) if cmp_f64 else float(thr))


def _valid(x, poff):
    return torch.from_numpy(np.stack([(~np.isnan(x[s:e])).sum(0) for s, e in O._groups(poff)]).astype(np.int32))


def to_time_cell(values, time_axis, device=None):
    a = _np(values)
    if time_axis != 0:
        a = np.moveaxis(a, time_axis, 0)
    a = np.ascontiguousarray(a, dtype=np.float32)
    return torch.from_numpy(a.reshape(a.shape[0], -1)), tuple(a.shape[1:])


def period_count(x2d, poff, op_code, thr, cmp_f64=False, want_valid=False):
    x = _np(x2d)
    out = np.stack([_cond(x[s:e], op_code, thr, cmp_f64).sum(0) for s, e in O._groups(poff)]).astype(np.int32)
    return torch.from_numpy(out), (_valid(x, poff) if want_valid else None)


def period_runstat(x2d, poff, op_code, thr, reducer_code, window, resample_before_rl=True, cmp_f64=False,
                   want_valid=False):
    x = _np(x2d)
    out = O.resample_and_rl(_cond(x, op_code, thr, cmp_f64), bool(resample_before_rl), O.rle_statistics, poff=poff,
                            reducer=RED_NAME[reducer_code], window=int(window))
    return torch.from_numpy(np.asarray(out, dtype=np.float32)), (_valid(x, poff) if want_valid else None)


def period_runstat_gap(x2d, poff, op_code, thr, reducer_code, min_gap, window=1, cmp_f64=False):
    x = _np(x2d)
    m = _cond(x, op_code, thr, cmp_f64)
    filled = O.runs_with_holes(m, 1, ~m, int(min_gap)).astype(np.float32)
    out = O.resample_and_rl(filled, True, O.rle_statistics, poff=poff, reducer=RED_NAME[reducer_code], window=window)
    return torch.from_numpy(np.asarray(out, dtype=np.float32))


def period_reduce(x2d, poff, stat_code, transform=0, op_code=0, thr=0.0, want_valid=False):
    x = _np(x2d)
    if transform == _lib.TF_EXCESS:
        out = O.cumulative_difference(x, float(thr), OP_NAME[op_code], poff)
    else:
        y = x.astype(np.float64)
        if transform == _lib.TF_WHERE:
            y = np.where(_cond(x, op_code, thr), y, np.nan)
        out = O.resample_reduce(y, poff, STAT_NAME[stat_code])
    return torch.from_numpy(np.asarray(out, dtype=np.float32)), (_valid(x, poff) if want_valid else None)


def rolling_period_reduce(x2d, poff, window, window_stat_code, center, stat_code):
    out = O.select_rolling_resample_op(_np(x2d).astype(np.float64), STAT_NAME[stat_code], int(window), poff,
                                       window_center=bool(center), window_op=STAT_NAME[window_stat_code])
    return torch.from_numpy(np.asarray(out, dtype=np.float32))


def rolling_period_reduce_sel(x2d, poff, window, window_stat_code, center, stat_code, keep):
    rolled = O.rolling(_np(x2d).astype(np.float64), int(window), STAT_NAME[window_stat_code], center=bool(center))
    rolled = np.where(np.asarray(keep, bool)[:, None], rolled, np.nan)
    return torch.from_numpy(np.asarray(O.resample_reduce(rolled, poff, STAT_NAME[stat_code]), dtype=np.float32))


def spell_runstat(x2d, poff, window, window_stat_code, op_code, thr, reducer_code, resample_before_rl=True):
    out = O.spell_length_statistics(_np(x2d), float(thr), int(window), STAT_NAME[window_stat_code], OP_NAME[op_code],
                                    RED_NAME[reducer_code], poff, resample_before_rl=bool(resample_before_rl))
    return torch.from_numpy(np.asarray(out, dtype=np.float32))


def period_run_maxsum(x2d, poff, op_code, thr, window, resample_before_rl=True):
    x = _np(x2d)
    t32 = np.float32(thr)
    excess = np.where(np.isnan(x), 0, np.clip((x - t32) if op_code in (0, 2) else (t32 - x), 0, None)).astype(np.float64)
    out = O.resample_and_rl(excess, bool(resample_before_rl), O.windowed_max_run_sum, int(window), poff=poff)
    return torch.from_numpy(np.asarray(out, dtype=np.float32))


def period_runstat2(x1, x2, poff, op1, thr1, op2, thr2, reducer_code, window, resample_before_rl=True, var_any=False):
    c1, c2 = _cond(_np(x1), op1, thr1), _cond(_np(x2), op2, thr2)
    m = (c1 | c2) if var_any else (c1 & c2)
    out = O.resample_and_rl(m, bool(resample_before_rl), O.rle_statistics, poff=poff, reducer=RED_NAME[reducer_code],
                            window=int(window))
    return torch.from_numpy(np.asarray(out, dtype=np.float32))


def percentile_doy(x2d, doy_index, year_index, n_doy, n_years, window, percentiles, alpha, beta, force_generic=False,
                   vrow=None):
    x = _np(x2d)
    if vrow is not None:
        vr = np.asarray(vrow)
        x = np.where((vr >= 0)[:, None], x[np.maximum(vr, 0)], np.nan).astype(np.float32)
    T, C = x.shape
    year, doy = np.asarray(year_index), np.asarray(doy_index)
    rr = O.rolling_construct_center(x, int(window))
    rrr = np.full((n_doy, n_years * window, C), np.nan, dtype=rr.dtype)
    for t in range(T):
        rrr[doy[t] - 1, year[t] * window:(year[t] + 1) * window] = rr[t]
    per = np.atleast_1d(np.asarray(percentiles, dtype=np.float64))
    out = np.stack([O.nan_quantile(rrr[d], per / 100.0, alpha, beta) for d in range(n_doy)])  # (n_doy, n_per, C)
    return torch.from_numpy(np.ascontiguousarray(np.moveaxis(out, 1, 0)))


def doy_interp(table2d, doy_min, doy_max):
    return torch.from_numpy(np.ascontiguousarray(O.interpolate_doy_calendar(_np(table2d), int(doy_max), int(doy_min))))


def doy_threshold_count(x2d, poff, doy_index, table2d, op_code, want_valid=False):
    x = _np(x2d)
    out = O.threshold_count(x, OP_NAME[op_code], _np(table2d)[np.asarray(doy_index) - 1], poff)
    return torch.from_numpy(np.asarray(out, dtype=np.int32)), (_valid(x, poff) if want_valid else None)


def mask_steps(x2d, keep):
    x = _np(x2d).copy()
    x[~np.asarray(keep, dtype=bool)] = np.nan
    return torch.from_numpy(x)


def period_boundary_run(x2d, poff, op_code, thr, window, last=False, cmp_f64=False):
    fn = O.last_run if last else O.first_run
    out = fn(_cond(_np(x2d), op_code, thr, cmp_f64), int(window), poff=poff)
    return torch.from_numpy(np.asarray(out, dtype=np.float32))


def period_boundary_run_range(x2d, poff, range_lo, range_hi, op_code, thr, window, last=False, negate=False,
                              cell_lo=None, cmp_f64=False):
    """Literal restatement of the C-ABI contract (include/xclim_b200.h, xc_period_boundary_run_range_f32):
    first / last run of >= window steps of the (optionally negated) condition inside
    [range_lo[p], range_hi[p]) of each period; window == 1 on the untouched whole period keeps the
    argmax == argmin rule."""
    x = _np(x2d)
    cond = _cond(x, op_code, thr, cmp_f64)
    if negate:
        cond = ~cond
    P, C = len(poff) - 1, x.shape[1]
    out = np.full((P, C), np.nan, dtype=np.float32)
    clo = None if cell_lo is None else _np(cell_lo)
    for p in range(P):
        t0, t1 = int(poff[p]), int(poff[p + 1])
        if int(range_lo[p]) < 0:
            continue
        for c in range(C):
            lo, hi = max(int(range_lo[p]), t0), min(int(range_hi[p]), t1)
            full = (lo == t0) and (hi == t1)
            if clo is not None:
                b = clo[p, c]
                bl = int(b) if b == b else 0
                if t0 + bl > lo:
                    lo, full = t0 + bl, False
            m = cond[lo:hi, c]
            if window == 1 and full:
                n = int(m.sum())
                if 0 < n < hi - lo:
                    idx = np.nonzero(m)[0]
                    out[p, c] = (idx[-1] if last else idx[0]) + lo - t0
                continue
            run = 0
            steps = range(hi - 1, lo - 1, -1) if last else range(lo, hi)
            for s in steps:
                run = run + 1 if cond[s, c] else 0
                if run >= window:
                    out[p, c] = (s + window - 1 - t0) if last else (s - window + 1 - t0)
                    break
    return torch.from_numpy(out)


def bootstrap_doy_count(x2d, base_start, n_base_years, year_len, step_period, P, window, percentile, alpha, beta,
                        op_code):
    """(P, C) float64: mean over the other base years of the in-base period counts; 0 for periods without
    base steps (the C-ABI contract of xc_bootstrap_doy_count_f32)."""
    x = _np(x2d)
    nb = n_base_years * year_len
    xb = x[base_start:base_start + nb]
    year = np.repeat(np.arange(n_base_years), year_len)
    doy = np.tile(np.arange(1, year_len + 1), n_base_years)
    sp = np.asarray(step_period)
    out = np.zeros((P, x.shape[1]))
    for y in range(n_base_years):
        rows = np.nonzero(year == y)[0]
        acc = {}
        for s_ in range(n_base_years):
            if s_ == y:
                continue
            z = xb.copy()
            z[rows] = xb[year == s_]
            tab = O.percentile_doy(z, year, doy, int(window), float(percentile), alpha, beta)[:, 0]
            hit = O.compare(xb[rows].astype(np.float64), OP_NAME[op_code], tab[doy[rows] - 1])
            for p in np.unique(sp[rows]):
                acc.setdefault(int(p), []).append(hit[sp[rows] == p].sum(0))
        for p, lst in acc.items():
            out[p] = np.mean(np.stack(lst), axis=0)
    return torch.from_numpy(out)


def eqm_train(ref2d, hist2d, nq, kind_code):
    af, hq = O.eqm_train(_np(ref2d), _np(hist2d), int(nq), "+" if kind_code == 0 else "*")
    return torch.from_numpy(np.ascontiguousarray(af, dtype=np.float32)), \
        torch.from_numpy(np.ascontiguousarray(hq, dtype=np.float32))


def eqm_adjust(sim2d, af, hq, kind_code, interp_code):
    out = O.eqm_adjust(_np(sim2d), _np(af), _np(hq), "+" if kind_code == 0 else "*",
                       "linear" if interp_code == 1 else "nearest")
    return torch.from_numpy(np.ascontiguousarray(out, dtype=np.float32))


def period_run_quantile(x2d, poff, op_code, thr, q, window, resample_before_rl=True, cmp_f64=False):
    out = O.resample_and_rl(_cond(_np(x2d), op_code, thr, cmp_f64), bool(resample_before_rl), O.rle_statistics,
                            poff=poff, reducer=float(q), window=int(window))
    return torch.from_numpy(np.asarray(out, dtype=np.float32))


def transpose_f64(m):
    return m.t().contiguous()


def table_cell_major(table):
    return table.permute(2, 1, 0).contiguous()


def spell_mask(x2d, window, window_stat_code, op_code, thr, keep=None, drop_nan_adjacent=False):
    """Oracle spell mask (oracle.spell_mask, indices/generic.py:503-535) + select_time + the two NaN rules."""
    x = _np(x2d)
    m = O.spell_mask(x, int(window), STAT_NAME[window_stat_code], OP_NAME[op_code], float(thr)).astype(np.float32)
    if keep is not None:
        keep = np.asarray(keep)
        if drop_nan_adjacent:
            for c in range(m.shape[1]):
                t = 0
                while t < m.shape[0]:
                    if keep[t] == 2 and m[t, c] > 0:
                        while t < m.shape[0] and keep[t] != 0 and m[t, c] > 0:
                            m[t, c] = 0
                            t += 1
                    else:
                        t += 1
        m[keep == 0] = np.nan
    return torch.from_numpy(m)


def period_count_arr(x2d, poff, op_code, thr2d, per_time):
    x = _np(x2d).astype(np.float64)
    t = _np(thr2d)
    with np.errstate(invalid="ignore"):
        cond = O.compare(x, OP_NAME[op_code], t if per_time else t[0][None, :])
    return torch.from_numpy(np.stack([cond[a:b].sum(0) for a, b in O._groups(poff)]).astype(np.int32))


def period_multi(x2d, poff, plan, n_slots):
    """Oracle composition of the fused multi-output pass (include/xclim_b200.h: XcMultiPlan)."""
    x = _np(x2d)
    P, C = len(poff) - 1, x.shape[1]
    out = np.zeros((max(1, n_slots), P, C), dtype=np.float32)
    groups = O._groups(poff)

    def put(slot, v, as_int=False):
        if slot >= 0:
            v = np.asarray(v)
            out[slot] = v.astype(np.int32).view(np.float32) if as_int else v.astype(np.float32)

    def run_stat(cond, red, w):
        return O.resample_and_rl(cond, True, O.rle_statistics, poff=poff, reducer=red, window=int(w))

    x64 = x.astype(np.float64)
    put(plan.slot_sum, O.resample_reduce(x64, poff, "sum"))
    put(plan.slot_mean, O.resample_reduce(x64, poff, "mean"))
    put(plan.slot_min, O.resample_reduce(x64, poff, "min"))
    put(plan.slot_max, O.resample_reduce(x64, poff, "max"))
    with np.errstate(invalid="ignore"):
        conds = []
        for j in range(plan.n_cond):
            e = plan.cond[j]
            cond = np.float32(e.sgn) * x > np.float32(e.thr)
            conds.append(cond)
            put(e.slot_n, np.stack([cond[a:b].sum(0) for a, b in groups]), True)
            m = run_stat(cond, "max", 1)
            put(e.slot_max, np.where(m >= e.wmax, m, 0))
        for k in range(plan.n_runs):
            r = plan.runs[k]
            assert r.cond == k // 2
            if r.slot >= 0:
                put(r.slot, run_stat(conds[r.cond], "sum" if r.kind == 0 else "count", r.window))
        for k in range(plan.n_msum):
            m = plan.msum[k]
            assert m.cond == 0
            exc = np.where(conds[m.cond], np.float32(m.sgn) * (x - np.float32(m.thr0)), np.float32(0)).astype(np.float64)
            put(m.slot, O.resample_and_rl(exc, True, O.windowed_max_run_sum, int(m.window), poff=poff))
        for j in range(plan.n_sums):
            e = plan.sums[j]
            if e.mode == 0:
                d = np.float32(e.off_sgn) * (x - np.float32(e.off))
                v = np.where(np.isnan(d), 0.0, np.maximum(d, np.float32(0)).astype(np.float64))
            else:
                v = np.where(np.float32(e.sgn) * x > np.float32(e.thr), x64, 0.0)
            put(e.slot, np.stack([v[a:b].sum(0) for a, b in groups]))
    return torch.from_numpy(out)


def dev_ints(arr, dtype, device):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(arr, dtype=dtype)))


def fire_weather(tas, pr, hurs, ws, snd, month, lat, season_mask, dc0, dmc0, ffmc0, winter_pr, outputs, params):
    """The oracle day loop behind the argument list of ``device.fire_weather`` (``params``: _lib.FwiParams)."""
    from oracle import fire_oracle as FO
    P = params
    season = {v: k for k, v in _lib.FWI_SEASONS.items()}[P.season_mode]
    dry = {v: k for k, v in _lib.FWI_DRY_STARTS.items()}[P.dry_start]
    ref = tas if tas is not None else pr
    T, C = ref.shape

    def series(x, i):
        if x is None:
            return np.full((T, C), np.nan, np.float32)
        return (_np(x).astype(np.float32) * np.float32(P.in_scale[i]) + np.float32(P.in_offset[i])).astype(np.float32)

    def state(x, fill):
        return np.full(C, fill, np.float32) if x is None else _np(x).astype(np.float32)

    codes = [o for o in outputs if o in FO._ORDER]
    full = FO.complete_indexes(codes) if codes else []
    extra = [o for o in outputs if o in ("season_mask", "winter_pr")]
    if P.season_mode >= 2 and "season_mask" not in extra:
        extra = extra + ["season_mask"]
    kw = dict(season_method=season, overwintering=bool(P.overwintering), dry_start=dry,
              initial_start_up=bool(P.initial_start_up), temp_start_thresh=P.temp_start_thresh,
              temp_end_thresh=P.temp_end_thresh, snow_thresh=P.snow_thresh, prec_thresh=P.prec_thresh,
              snow_min_mean_depth=P.snow_min_mean_depth, dc_start=P.dc_start, dmc_start=P.dmc_start,
              ffmc_start=P.ffmc_start, dc_dry_factor=P.dc_dry_factor, dmc_dry_factor=P.dmc_dry_factor,
              snow_min_cover_frac=P.snow_min_cover_frac, carry_over_fraction=P.carry_over_fraction,
              wetting_efficiency_fraction=P.wetting_efficiency_fraction,
              temp_condition_days=P.temp_condition_days, snow_condition_days=P.snow_condition_days,
              snow_cover_days=P.snow_cover_days)
    lat_h = np.zeros(C) if lat is None else np.asarray(lat, dtype=np.float64)
    mask = None if season_mask is None else _np(season_mask).astype(bool)
    res = FO.fire_weather_calc(series(tas, 0), series(pr, 1), series(hurs, 2), series(ws, 3), series(snd, 4),
                               np.asarray(month), lat_h, mask, state(dc0, np.nan), state(dmc0, np.nan),
                               state(ffmc0, np.nan), state(winter_pr, 0.0), outputs=full + extra, **kw)
    out = {}
    for name in outputs:
        a = np.asarray(res[name])
        out[name] = torch.from_numpy(np.ascontiguousarray(a.astype(np.uint8) if name == "season_mask" else a))
    return out


def to_device_f32(values):
    return torch.from_numpy(np.ascontiguousarray(_np(values), dtype=np.float32))


def fire_elementwise(kind, a, b=None, p=(0.0, 0.0, 0.0)):
    from oracle import fire_oracle as FO
    x, y = _np(a).astype(np.float32), (None if b is None else _np(b).astype(np.float32))
    if kind == "OWDC":
        r = FO.overwintering_drought_code(x, y, *p)
    else:
        fn = {"ISI": FO.initial_spread_index, "BUI": FO.build_up_index, "FWI": FO.fire_weather_index,
              "DSR": FO.daily_severity_rating}[kind]
        r = fn(x) if y is None else fn(x, y)
    return torch.from_numpy(np.ascontiguousarray(np.asarray(r, dtype=np.float32)))


FUNCTIONS = [to_time_cell, period_count, period_runstat, period_runstat_gap, period_reduce, rolling_period_reduce,
             spell_runstat, period_run_maxsum, period_runstat2, percentile_doy, doy_interp, doy_threshold_count,
             mask_steps, dev_ints, period_boundary_run, period_boundary_run_range, bootstrap_doy_count, eqm_train,
             eqm_adjust, period_run_quantile, table_cell_major, period_multi, period_count_arr, spell_mask, transpose_f64,
             rolling_period_reduce_sel, fire_weather, fire_elementwise, to_device_f32]


def install(monkeypatch):
    from xclim_b200 import device
    for fn in FUNCTIONS:
        monkeypatch.setattr(device, fn.__name__, fn)
