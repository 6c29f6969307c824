"""GPU parity of the day-of-year table kernels (WSDI / CSDI run statistics, the R95pTOT sums, the compound
percentile days) and the daily temperature range kernel against the oracle: every period kind, both
resample_before_rl modes, every operator, three calendars with tables of another length, the vec4 and scalar paths
(C % 4 != 0, ldx != C, C just above a block multiple), the indicator level and the streamed host path."""
import numpy as np
import pytest

from oracle import etccdi_oracle as E
from oracle import xclim_oracle as O
from xb_helpers import make_field

pytestmark = pytest.mark.gpu

FREQS = ("YS", "MS", "QS-DEC", "YS-JUL")
OPS = (">", ">=", "<", "<=")


def _series(rng, T, C, base=280.0, amp=8.0):
    t = np.arange(T)[:, None]
    x = base + amp * np.sin(2 * np.pi * t / 365.0) + 3 * rng.standard_normal((T, C))
    x = x.astype(np.float32)
    x[rng.random(x.shape) < 0.01] = np.nan
    return x


def _table_like(rng, x, n_doy, doy):
    """A float64 per-doy table near the data, with entries equal to float32 data values (ties) and values between
    two float32s (the float64 compare matters)."""
    C = x.shape[1]
    tab = np.full((n_doy, C), np.nan)
    for d in range(1, n_doy + 1):
        rows = np.nonzero(doy == d)[0]
        if rows.size:
            tab[d - 1] = np.nan_to_num(x[rows[0]].astype(np.float64), nan=280.0)
    tab = np.where(np.isnan(tab), 280.0, tab)
    tab += np.where(rng.random(tab.shape) < 0.5, 0.0, rng.standard_normal(tab.shape) * 1e-6)
    return tab


def _views(rng, x, C):
    """(name, device (T, C) view): contiguous, and a column slice of a wider buffer (ldx != C)."""
    import torch
    T = x.shape[0]
    wide = torch.full((T, C + 5), float("nan"), device="cuda")
    wide[:, 1:C + 1] = torch.from_numpy(x).cuda()
    return [("contiguous", torch.from_numpy(x).cuda()), ("ldx", wide[:, 1:C + 1])]


@pytest.mark.parametrize("calendar", ["noleap", "360_day", "standard"])
@pytest.mark.parametrize("C", [8, 131, 516])
def test_doy_runstat_kernel(cuda, calendar, C):
    import torch

    from xclim_b200 import TimeAxis, _lib, device
    rng = np.random.default_rng(C)
    T = {"noleap": 365, "360_day": 360, "standard": 365}[calendar] * 4 + 40
    ta = TimeAxis.daily("2001-03-01", T, calendar)
    doy = np.asarray(ta.doy)
    x = _series(rng, T, C)
    n_doy = int(ta.max_doy)
    tab = _table_like(rng, x, n_doy, doy)
    tab_d = torch.from_numpy(tab).cuda()
    cases = [(">", "sum", 6), ("<", "sum", 3), (">=", "max", 1), ("<=", "count", 40), (">", "mean", 2),
             ("<", "std", 1), (">=", "min", 2)]
    for freq in FREQS:
        poff = ta.period_offsets(freq)
        for op, red, w in cases:
            cond = O.compare(x, op, tab[doy - 1])
            for rbrl in (True, False):
                exp = O.resample_and_rl(cond, rbrl, O.rle_statistics, poff=poff, reducer=red, window=w)
                for name, xv in _views(rng, x, C):
                    got, valid = device.doy_runstat(xv, poff, doy, tab_d, _lib.OPS[op], _lib.RL_REDUCERS[red], w,
                                                    rbrl, want_valid=True)
                    np.testing.assert_array_equal(got.cpu().numpy(), np.asarray(exp, np.float32),
                                                  err_msg=f"{freq} {op} {red} w={w} rbrl={rbrl} {name}")
                    np.testing.assert_array_equal(valid.cpu().numpy(),
                                                  np.stack([(~np.isnan(x[s:e])).sum(0) for s, e in O._groups(poff)]))


@pytest.mark.parametrize("calendar,n_doy", [("noleap", 366), ("360_day", 365), ("standard", 365)])
def test_spell_duration_indices_other_table_length(cuda, calendar, n_doy):
    from xclim_b200 import indices
    rng = np.random.default_rng(n_doy)
    T = 3 * (360 if calendar == "360_day" else 365) + 100
    x = _series(rng, T, 36).reshape(T, 6, 6)
    da = make_field(x, "2000-02-01", calendar=calendar, units="K")
    tab = 280 + 3 * rng.standard_normal((n_doy, 36))
    from test_etccdi_cpu import _per_field
    per = _per_field(tab.reshape(n_doy, 6, 6), "K", ("d0", "d1"))
    cal_max = int(da.time.max_doy)
    doy = np.asarray(da.time.doy)
    for freq in ("YS", "MS"):
        poff = da.time.period_offsets(freq)
        for rbrl in (True, False):
            got = indices.warm_spell_duration_index(da, per, window=4, freq=freq, resample_before_rl=rbrl)
            exp = E.warm_spell_duration_index(x, tab.reshape(n_doy, 6, 6), doy, poff, 4, rbrl, ">", cal_max)
            np.testing.assert_array_equal(got.values, exp)
            got = indices.cold_spell_duration_index(da, per, window=2, freq=freq, resample_before_rl=rbrl, op="<=")
            exp = E.cold_spell_duration_index(x, tab.reshape(n_doy, 6, 6), doy, poff, 2, rbrl, "<=", cal_max)
            np.testing.assert_array_equal(got.values, exp)


@pytest.mark.parametrize("C", [8, 131, 516])
def test_sums_kernel(cuda, C):
    import torch

    from xclim_b200 import TimeAxis, _lib, device
    rng = np.random.default_rng(7 + C)
    ta = TimeAxis.daily("2001-01-01", 365 * 3, "noleap")
    doy = np.asarray(ta.doy)
    T = len(ta)
    x = (rng.gamma(0.6, 5.0, (T, C)) * (rng.random((T, C)) < 0.6)).astype(np.float32)
    x[rng.random(x.shape) < 0.01] = np.nan
    x[rng.random(x.shape) < 0.02] = 1.0                       # days at the wet-day threshold
    tab = _table_like(rng, np.where(x > 1, x, 5.0).astype(np.float32), 365, doy)
    per_cell = rng.gamma(2.0, 3.0, (1, C))
    for freq in FREQS:
        poff = ta.period_offsets(freq)
        for op in (">", ">="):
            for name, xv in _views(rng, x, C):
                for table, idx in ((tab, doy), (per_cell, None)):
                    s_thr, s_wet = device.period_sums_thr(xv, poff, _lib.OPS[op], torch.from_numpy(table).cuda(), 1.0,
                                                          doy_index=idx)
                    tp = table[doy - 1] if idx is not None else np.broadcast_to(table, x.shape)
                    over = np.where(O.compare(x, op, tp), x, 0)
                    wet = np.where(O.compare(x, op, 1.0), x, 0)
                    for got, a in ((s_thr, over), (s_wet, wet)):
                        exp = np.stack([a[s:e].sum(0, dtype=np.float64) for s, e in O._groups(poff)]).astype(np.float32)
                        np.testing.assert_allclose(got.cpu().numpy(), exp, rtol=1e-6, atol=0,
                                                   err_msg=f"{freq} {op} {name} doy={idx is not None}")


def test_fraction_over_precip_thresh_end_to_end(cuda):
    from xclim_b200 import TimeAxis, indices
    rng = np.random.default_rng(11)
    ta = TimeAxis.daily("2000-01-01", 366 + 365 * 2, "standard")
    T = len(ta)
    x = (rng.gamma(0.6, 5.0, (T, 4, 5)) * (rng.random((T, 4, 5)) < 0.5)).astype(np.float32)
    x[:, 0, 0] = 0                                                  # no wet day: NaN
    pr = make_field(x, "2000-01-01", calendar="standard", units="mm/d")
    tab = rng.gamma(2.0, 4.0, (365, 4, 5))
    tab[::7, 1] = np.nan
    from test_etccdi_cpu import _per_field
    per = _per_field(tab, "mm/d", ("d0", "d1"))
    for freq in ("YS", "MS"):
        got = indices.fraction_over_precip_thresh(pr, per, thresh="1 mm/d", freq=freq)
        exp = E.fraction_over_precip_thresh(x, tab, 1.0, pr.time.period_offsets(freq), doy=np.asarray(pr.time.doy),
                                            cal_max_doy=366)
        np.testing.assert_array_equal(np.isnan(got.values), np.isnan(exp))
        np.testing.assert_allclose(got.values, exp, rtol=2e-6)
        assert np.isnan(got.values[:, 0, 0]).all()


@pytest.mark.parametrize("C", [8, 131, 516])
def test_count2_kernel(cuda, C):
    import torch

    from xclim_b200 import TimeAxis, _lib, device
    rng = np.random.default_rng(21 + C)
    ta = TimeAxis.daily("2001-01-01", 360 * 3 + 17, "360_day")
    doy = np.asarray(ta.doy)
    T = len(ta)
    t = _series(rng, T, C)
    p = (rng.gamma(0.7, 3.0, (T, C))).astype(np.float32)
    p[rng.random(p.shape) < 0.01] = np.nan
    tt = _table_like(rng, t, 360, doy)
    pt = _table_like(rng, p, 360, doy)
    tt_d, pt_d = torch.from_numpy(tt).cuda(), torch.from_numpy(pt).cuda()
    for op1 in OPS:
        for op2 in OPS:
            c = O.compare(t, op1, tt[doy - 1]) & O.compare(p, op2, pt[doy - 1])
            for freq in FREQS:
                poff = ta.period_offsets(freq)
                exp = np.stack([c[s:e].sum(0) for s, e in O._groups(poff)]).astype(np.float32)
                for (name, tv), (_, pv) in zip(_views(rng, t, C), _views(rng, p, C)):
                    got = device.doy_count2(tv, pv, poff, doy, tt_d, pt_d, _lib.OPS[op1], _lib.OPS[op2])
                    np.testing.assert_array_equal(got.cpu().numpy(), exp, err_msg=f"{op1} {op2} {freq} {name}")


@pytest.mark.parametrize("name", sorted(E._COMPOUND))
def test_compound_indices_mixed_table_calendars(cuda, name):
    """A 366-day temperature table and a 365-day precipitation table against noleap data that starts in March."""
    from xclim_b200 import indices
    rng = np.random.default_rng(len(name))
    T = 365 * 2
    t = _series(rng, T, 12).reshape(T, 3, 4)
    p = rng.gamma(0.7, 3.0, (T, 3, 4)).astype(np.float32)
    tas = make_field(t, "2001-03-01", calendar="noleap", units="K")
    pr = make_field(p, "2001-03-01", calendar="noleap", units="mm/d")
    tt = 280 + 3 * rng.standard_normal((366, 3, 4))
    pt = rng.gamma(1.0, 2.0, (365, 3, 4))
    from test_etccdi_cpu import _per_field
    got = getattr(indices, name)(tas, pr, _per_field(tt, "K", ("d0", "d1")), _per_field(pt, "mm/d", ("d0", "d1")),
                                 freq="MS")
    exp = E.compound_days(name, t, p, tt, pt, np.asarray(tas.time.doy), tas.time.period_offsets("MS"), 365)
    np.testing.assert_array_equal(got.values, exp)


@pytest.mark.parametrize("C", [8, 131, 516])
def test_range_stat_kernel(cuda, C):
    from xclim_b200 import TimeAxis, _lib, device
    rng = np.random.default_rng(31 + C)
    ta = TimeAxis.daily("2000-01-01", 366 + 365 + 45, "standard")
    T = len(ta)
    lo = _series(rng, T, C)
    hi = (lo + rng.uniform(0, 15, lo.shape)).astype(np.float32)
    for freq in FREQS:
        poff = ta.period_offsets(freq)
        for (name, lv), (_, hv) in zip(_views(rng, lo, C), _views(rng, hi, C)):
            for op in ("mean", "min", "max", "std", "sum", "var"):
                got = device.period_range_stat(lv, hv, poff, _lib.STATS[op]).cpu().numpy()
                exp = E.daily_temperature_range(lo, hi, poff, op)
                if op in ("min", "max"):
                    np.testing.assert_array_equal(got, exp, err_msg=f"{op} {freq} {name}")
                else:
                    np.testing.assert_allclose(got, exp, rtol=2e-6, atol=2e-5, err_msg=f"{op} {freq} {name}")
            got = device.period_range_stat(lv, hv, poff, _lib.STATS["mean"], variability=True).cpu().numpy()
            np.testing.assert_allclose(got, E.daily_temperature_range_variability(lo, hi, poff), rtol=2e-6,
                                       err_msg=f"variability {freq} {name}")


def test_indicators_mask_missing_days(cuda):
    from xclim_b200 import atmos
    rng = np.random.default_rng(41)
    T = 365 * 2
    x = _series(rng, T, 6)
    x[:] = np.where(np.isnan(x), 280, x)
    x[40, 2] = np.nan
    tx = make_field(x, "2001-01-01", calendar="noleap", units="K")
    from test_etccdi_cpu import _per_field
    per = _per_field(280 + 3 * rng.standard_normal((365, 6)), "K")
    out = atmos.warm_spell_duration_index(tx, per, window=2, freq="MS").values
    assert np.isnan(out[1, 2]) and np.isfinite(np.delete(out, 2, axis=1)).all() and np.isfinite(out[0, 2])
    p = rng.gamma(0.7, 3.0, (T, 6)).astype(np.float32)
    pr = make_field(p, "2001-01-01", calendar="noleap", units="mm/d")
    out = atmos.warm_and_wet_days(tx, pr, per, _per_field(np.ones((365, 6)), "mm/d"), freq="MS").values
    assert np.isnan(out[1, 2]) and np.isfinite(out[2, 2])
    out = atmos.daily_temperature_range(tx, tx, freq="MS").values
    assert np.isnan(out[1, 2]) and out[1, 1] == 0


def test_streamed_host_inputs_match_device_resident(cuda):
    import torch

    import xclim_b200
    from xclim_b200 import Field, TimeAxis, indices
    rng = np.random.default_rng(51)
    ta = TimeAxis.daily("2001-01-01", 365 * 2, "noleap")
    T, nl, nx = len(ta), 9, 8
    t = _series(rng, T, nl * nx).reshape(T, nl, nx)
    p = rng.gamma(0.7, 3.0, (T, nl, nx)).astype(np.float32)
    tt = np.ascontiguousarray(np.moveaxis(280 + 3 * rng.standard_normal((365, nl, nx)), 0, -1))
    pt = np.ascontiguousarray(np.moveaxis(rng.gamma(1.0, 2.0, (365, nl, nx)), 0, -1))

    def f(v, u):
        return Field(v, ("time", "lat", "lon"), ta, {}, {"units": u})

    def per(v, u):
        return Field(v, ("lat", "lon", "dayofyear"), None, {"dayofyear": np.arange(1, 366)}, {"units": u})

    calls = [
        ("warm_spell_duration_index", lambda a, b: indices.warm_spell_duration_index(a["t"], per(tt, "K"), freq="MS")),
        ("fraction_over_precip_thresh", lambda a, b: indices.fraction_over_precip_thresh(a["p"], per(pt, "mm/d"))),
        ("cold_and_wet_days", lambda a, b: indices.cold_and_wet_days(a["t"], a["p"], per(tt, "K"), per(pt, "mm/d"))),
        ("daily_temperature_range_variability",
         lambda a, b: indices.daily_temperature_range_variability(a["t"], a["t2"], freq="QS-DEC")),
    ]
    host = {"t": f(t, "K"), "p": f(p, "mm/d"), "t2": f((t + 7).astype(np.float32), "K")}
    dev = {k: Field(torch.from_numpy(np.asarray(v.values)).cuda(), v.dims, ta, {}, dict(v.attrs)) for k, v in host.items()}
    for name, call in calls:
        with xclim_b200.set_options(stream_min_bytes=1, stream_slab_bytes=T * nx * 4 * 2):
            streamed = call(host, None)
        with xclim_b200.set_options(device_outputs=True):
            resident = call(dev, None)
        r = resident.values.cpu().numpy() if hasattr(resident.values, "cpu") else np.asarray(resident.values)
        np.testing.assert_array_equal(np.asarray(streamed.values), r, err_msg=name)
        assert streamed.dims == ("time", "lat", "lon")
