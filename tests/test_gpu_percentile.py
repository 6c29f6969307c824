"""GPU parity: percentile_doy (generic + fast kernels), doy interpolation, tx90p counts."""
import numpy as np
import pytest

from oracle import xclim_oracle as O
from xb_helpers import make_field, plant_infinite_samples

pytestmark = pytest.mark.gpu

RTOL = 1e-5  # north_star tolerance for float percentile outputs (observed: bit-identical)


def _tas(rng, T, shape, nan_frac=0.01):
    t = np.arange(T)
    x = 288 + 12 * np.sin(2 * np.pi * (t % 365 - 110) / 365)[(slice(None),) + (None,) * len(shape)]
    x = x + 3 * rng.standard_normal((T,) + shape)
    x = x.astype(np.float32)
    x[rng.random(x.shape) < nan_frac] = np.nan
    return x


def _table(per_field):
    """(n_doy, *space) from the reference-ordered (*space, dayofyear, percentiles) output."""
    v = per_field.values
    return np.moveaxis(v[..., 0], -1, 0)


@pytest.mark.parametrize("calendar,years", [("noleap", 6), ("noleap", 30), ("360_day", 4)])
@pytest.mark.parametrize("per", [90.0, 10.0, 99.0])
def test_percentile_doy_uniform_calendars(cuda, calendar, years, per):
    from xclim_b200 import calendar as xcal, device, TimeAxis
    rng = np.random.default_rng(11)
    L = 365 if calendar == "noleap" else 360
    T = years * L
    shape = (5, 9)
    x = _tas(rng, T, shape)
    x[:, 0, 0] = np.nan          # an all-NaN cell
    x[5:400, 0, 1] = np.nan      # a long gap
    plant_infinite_samples(x, [per / 100], range(40, 45), seed=years)
    da = make_field(x, "1981-01-01", calendar=calendar, units="K")
    got = xcal.percentile_doy(da, window=5, per=per)
    exp = O.percentile_doy(x, da.time.year, da.time.doy, 5, per)[:, 0]
    assert got.dims[-2:] == ("dayofyear", "percentiles") and got.values.dtype == np.float64
    np.testing.assert_allclose(_table(got), exp, rtol=RTOL, equal_nan=True)
    np.testing.assert_array_equal(_table(got), exp)  # in fact bit-identical (same lerp, same rounding)
    assert got.attrs["climatology_bounds"][0] == "1981-01-01" and got.attrs["window"] == 5
    assert "percentile_doy" in got.attrs["history"] and got.attrs["units"] == "K"
    # the fast and the generic kernels agree bit for bit
    import torch
    xd = torch.from_numpy(x.reshape(T, -1)).cuda()
    yidx = (np.arange(T) // L).astype(np.int16)
    a = device.percentile_doy(xd, da.time.doy, yidx, L, years, 5, [per], 1 / 3, 1 / 3)
    b = device.percentile_doy(xd, da.time.doy, yidx, L, years, 5, [per], 1 / 3, 1 / 3, force_generic=True)
    assert torch.equal(torch.nan_to_num(a, nan=-1.0), torch.nan_to_num(b, nan=-1.0))


@pytest.mark.parametrize("window", [1, 3, 5, 7, 9])
def test_percentile_doy_windows_and_types(cuda, window):
    from xclim_b200 import calendar as xcal
    rng = np.random.default_rng(12)
    x = _tas(rng, 365 * 8, (4, 4))
    plant_infinite_samples(x, [0.05, 0.95], range(6, 16), seed=window)
    da = make_field(x, "1990-01-01", calendar="noleap", units="K")
    for alpha, beta in ((1 / 3, 1 / 3), (1.0, 1.0), (0.0, 1.0)):
        got = xcal.percentile_doy(da, window=window, per=[5.0, 95.0], alpha=alpha, beta=beta)
        exp = O.percentile_doy(x, da.time.year, da.time.doy, window, [5.0, 95.0], alpha, beta)
        np.testing.assert_array_equal(np.moveaxis(got.values, (-2, -1), (0, 1)), exp)
    with pytest.raises(NotImplementedError):
        xcal.percentile_doy(da, window=4)


def test_percentile_doy_standard_calendar_and_366(cuda):
    """Leap years: generic kernel + the 1..365 -> 1..366 re-interpolation (core/calendar.py:484-485)."""
    from xclim_b200 import calendar as xcal
    rng = np.random.default_rng(13)
    T = 365 * 9 + 2
    x = _tas(rng, T, (3, 5))
    da = make_field(x, "1999-01-01", calendar="standard", units="K")
    got = xcal.percentile_doy(da, window=5, per=90.0)
    exp = O.percentile_doy(x, da.time.year, da.time.doy, 5, 90.0)[:, 0]
    assert _table(got).shape[0] == 366
    # the re-interpolation (xc_doy_interp_f64) repeats np.interp's operations: bit-identical
    np.testing.assert_array_equal(_table(got), exp)
    # partial first/last years (series not starting on Jan 1st)
    da2 = make_field(x[100:-50], "1999-04-11", calendar="standard", units="K")
    got2 = xcal.percentile_doy(da2, window=5, per=10.0)
    exp2 = O.percentile_doy(x[100:-50], da2.time.year, da2.time.doy, 5, 10.0)[:, 0]
    np.testing.assert_array_equal(_table(got2), exp2)


def test_percentile_doy_reference_known_answers(cuda):
    from xclim_b200 import calendar as xcal
    # tests/test_calendar.py:83-103
    tas = make_field(np.arange(365, dtype=np.float32), "2001-01-01", units="K")
    p1 = xcal.percentile_doy(tas, window=5, per=50)
    assert _table(p1)[2] == 2 and p1.attrs["units"] == "K"
    v = np.arange(365, dtype=np.float32); v[1] = np.nan
    pn = xcal.percentile_doy(make_field(v, "2001-01-01", units="K"), window=5, per=50)
    assert _table(pn)[2] == 2.5


def test_tx90p_counts(cuda):
    from xclim_b200 import calendar as xcal, indices
    rng = np.random.default_rng(14)
    years = 12
    x = _tas(rng, 365 * years, (6, 10))
    da = make_field(x, "1981-01-01", calendar="noleap", units="K")
    per = xcal.select_percentile(xcal.percentile_doy(da, window=5, per=90.0), 90.0)
    tab = O.percentile_doy(x, da.time.year, da.time.doy, 5, 90.0)[:, 0]
    for freq in ("YS", "MS"):
        for op in (">", ">="):
            got = indices.tx90p(da, per, freq=freq, op=op)
            exp = O.doy_threshold_count(x, tab, da.time.doy, da.time.period_offsets(freq), op)
            assert got.values.dtype == np.int64 and got.attrs["units"] == "d"
            np.testing.assert_array_equal(got.values, exp)
    per10 = xcal.select_percentile(xcal.percentile_doy(da, window=5, per=10.0), 10.0)
    tab10 = O.percentile_doy(x, da.time.year, da.time.doy, 5, 10.0)[:, 0]
    np.testing.assert_array_equal(indices.tx10p(da, per10, freq="YS").values,
                                  O.doy_threshold_count(x, tab10, da.time.doy, da.time.period_offsets("YS"), "<"))
    with pytest.raises(ValueError, match="not permitted"):
        indices.tx90p(da, per, op="<")
    # a percentile array handed over as plain host data (no cached device table) gives the same counts
    from xclim_b200 import Field
    per_host = Field(np.array(per.values, copy=True), per.dims, None, dict(per.coords), dict(per.attrs))
    np.testing.assert_array_equal(indices.tx90p(da, per_host, freq="YS").values,
                                  indices.tx90p(da, per, freq="YS").values)


def test_tx90p_reference_known_answer_leap_year(cuda):
    """tests/test_indices.py:2594-2607 (366-day year, per=10): monthly counts 30, 29, ..., 25."""
    from xclim_b200 import calendar as xcal, indices
    tas = np.arange(366, dtype=np.float32)
    da = make_field(tas, "2000-01-01", units="K")
    t90 = xcal.select_percentile(xcal.percentile_doy(da, per=10), 10.0)
    tas2 = tas.copy(); tas2[175:180] = 1
    out = indices.tx90p(make_field(tas2, "2000-01-01", units="K"), t90, freq="MS")
    assert out.values[0] == 30 and out.values[1] == 29 and out.values[5] == 25


@pytest.mark.parametrize("op", [">", ">=", "<", "<=", "==", "!="])
def test_doy_count_year_blocked_kernel_exact_ties(cuda, op):
    """Every float64-threshold count folds its thresholds to float32 by directed rounding (fold_f64): it must
    agree with the float64 compare for thresholds equal to data values, one double-ulp off, +-0, inf, NaN --
    through every threshold source (year-blocked table, day-of-year table with 4 and with 1 cell per thread,
    per-cell and per-step arrays) and every way to the 1-cell layout (C % 4 != 0, ldx > C, a base pointer
    one float off).  == and != have no year-blocked kernel: their yearly count takes the day-of-year kernel."""
    import torch
    from xclim_b200 import device, _lib
    rng = np.random.default_rng(15)
    L, N, C = 365, 7, 64
    x = (np.round(rng.standard_normal((L * N, C)) * 4) / 4).astype(np.float32)
    x[rng.random(x.shape) < 0.01] = np.nan
    tab = x[:L].astype(np.float64).copy()                       # exact ties with year 0
    tab[1::3] = np.nextafter(tab[1::3], np.inf)                 # just above a representable value
    tab[2::3] = np.nextafter(tab[2::3], -np.inf)                # just below
    tab[5, :8] = [0.0, -0.0, np.inf, -np.inf, np.nan, 1e-300, -1e-300, 1e300]
    x[5, :8] = [0.0, -0.0, 1.0, -1.0, 0.0, 0.0, -0.0, 3e38]
    poff = np.arange(N + 1, dtype=np.int32) * L
    month = np.concatenate([[0], np.cumsum(np.tile([31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31], N))]).astype(np.int32)
    doy = np.tile(np.arange(1, L + 1), N).astype(np.int16)
    code = _lib.OPS[op]
    xd, td = torch.from_numpy(x).cuda(), torch.from_numpy(tab).cuda()

    def expect(thr, po, cols=slice(None)):
        return O.threshold_count(x[:, cols], op, thr, po, constrain=[op])

    def nvalid(po, cols=slice(None)):
        return np.stack([(~np.isnan(x[s:e, cols])).sum(0) for s, e in zip(po[:-1], po[1:])])

    def check(got, exp):
        np.testing.assert_array_equal(got.cpu().numpy(), exp)

    for po in (poff, month):                 # yearly: year-blocked (inequalities); monthly: 4 cells per thread
        got, valid = device.doy_threshold_count(xd, po, doy, td, code, want_valid=True)
        check(got, expect(tab[doy - 1], po))
        check(valid, nvalid(po))
    # the 1-cell layouts: an odd number of cells, a row stride of 65 floats, a base pointer 4 bytes past 16-byte alignment
    wide = torch.full((L * N, 65), 9.0, dtype=torch.float32, device="cuda")
    wide[:, :64] = xd
    shifted = torch.full((L * N, 68), 9.0, dtype=torch.float32, device="cuda")
    shifted[:, 1:65] = xd
    layouts = [(xd[:, :63].contiguous(), slice(0, 63)), (wide[:, :64], slice(None)),
               (shifted[:, 1:65], slice(None))]
    assert layouts[1][0].stride(0) == 65 and layouts[2][0].data_ptr() % 16 == 4
    for xv, cols in layouts:
        tv = td[:, cols].contiguous()
        for po in (poff, month):
            got, valid = device.doy_threshold_count(xv, po, doy, tv, code, want_valid=True)
            check(got, expect(tab[doy - 1][:, cols], po, cols))
            check(valid, nvalid(po, cols))
        # array thresholds: per step (T, C) and per cell (1, C), the latter from the rows holding the edge values
        tstep = torch.from_numpy(tab[doy - 1][:, cols].copy()).cuda()
        check(device.period_count_arr(xv, month, code, tstep, True), expect(tab[doy - 1][:, cols], month, cols))
        for r in (5, 1, 2):
            tcell = torch.from_numpy(tab[r:r + 1, cols].copy()).cuda()
            check(device.period_count_arr(xv, month, code, tcell, False), expect(tab[r, cols], month, cols))
    # the array thresholds with 4 cells per thread
    check(device.period_count_arr(xd, poff, code, torch.from_numpy(tab[doy - 1].copy()).cuda(), True),
          expect(tab[doy - 1], poff))
    check(device.period_count_arr(xd, month, code, td[5:6].contiguous(), False), expect(tab[5], month))


@pytest.mark.parametrize("calendar,years,window", [("noleap", 30, 5), ("standard", 20, 9), ("360_day", 40, 5)])
def test_percentile_doy_mid_percentiles_selection_kernel(cuda, calendar, years, window):
    """Percentiles whose order statistics are more than 64 ranks from both ends of the sample (the
    median of 150 values ...) go through the selection kernel; a list of percentiles mixes it with the
    network kernels.  Heavy ties, NaNs, an all-NaN cell, a single-value cell and infinite samples included."""
    from xclim_b200 import calendar as xcal
    rng = np.random.default_rng(13)
    L = {"noleap": 365, "standard": 365.25, "360_day": 360}[calendar]
    T = int(years * L)
    x = _tas(rng, T, (6, 5), nan_frac=0.02)
    if calendar != "standard":   # (the 365 -> 366 re-interpolation of such tables is not covered here)
        plant_infinite_samples(x, [0.5, 0.1, 0.9], range(15, 30), seed=years)
    x[:, 0, 0] = np.nan
    x[:, 0, 1] = np.round(x[:, 0, 1])            # ties
    x[:, 0, 2] = np.where(rng.random(T) < 0.5, 0.0, -0.0).astype(np.float32)  # signed zeros only
    x[:, 1, 0] = np.nan
    x[100, 1, 0] = 7.0                            # one valid value in the whole series
    da = make_field(x, "1981-01-01", calendar=calendar, units="K")
    pers = [50.0, 10.0, 42.0, 90.0, 58.5]
    got = xcal.percentile_doy(da, window=window, per=pers)
    exp = O.percentile_doy(x, da.time.year, da.time.doy, window, pers)       # (n_doy, n_per, *space)
    g = np.moveaxis(got.values, (-2, -1), (0, 1))
    assert g.shape == exp.shape
    np.testing.assert_allclose(g, exp, rtol=RTOL, equal_nan=True)
    np.testing.assert_array_equal(g, exp)


@pytest.mark.parametrize("per,years", [(90.0, 30), (90.0, 31), (92.0, 32), (10.0, 30), (10.0, 31), (8.0, 32)])
def test_percentile_doy_tma_path(cuda, years, per, monkeypatch):
    """The TMA-fed window-5 kernel (30..32 uniform years, ldx % 4 == 0): bit-exact vs the oracle and vs
    the lane-by-lane kernel, with NaNs, infinities of both signs (the FADD NaN probe's false positive),
    cells beyond the last full 128-cell tile, windows that reach into the neighbouring year, and samples
    whose interpolation meets infinities or overflows (NaN lerp -> the sample maximum).  32 years take
    the 92nd / 8th percentile: the 90th / 10th need 17 order statistics there, beyond the TMA kernel's 16."""
    import torch
    from dispatch_host_build import pdoy_kernels as kernels
    from xclim_b200 import device
    rng = np.random.default_rng(100 + years)
    L, T = 365, years * 365
    shape = (4, 35)                       # 140 cells: one full TMA tile + a partial one
    x = _tas(rng, T, shape, nan_frac=0.002)
    x[:, 0, 0] = np.nan
    x[100:900, 0, 1] = np.nan
    x[7, 1, 2], x[365 + 7, 1, 2] = np.inf, -np.inf        # same day of year: inf + (-inf) = NaN in the probe
    x[0:3, 2, 3] = np.nan                                 # first days of the series
    x[T - 2:, 2, 4] = np.nan                              # last days
    plant_infinite_samples(x, [per / 100], list(range(60, 63)) + [138, 139], seed=years)
    doy = (np.arange(T) % L + 1).astype(np.int16)
    yidx = (np.arange(T) // L).astype(np.int16)
    xd = torch.from_numpy(x.reshape(T, -1)).cuda()
    assert xd.shape[1] % 4 == 0
    C = xd.shape[1]
    assert kernels(doy, yidx, L, years, 5, [per], C) == {f"w5t<{years - 16}>"}
    assert kernels(doy, yidx, L, years, 5, [per], C, no_tma=True) == {"w5p<16, false>"}
    monkeypatch.delenv("XCLIM_B200_NO_TMA", raising=False)
    a = device.percentile_doy(xd, doy, yidx, L, years, 5, [per], 1 / 3, 1 / 3)
    monkeypatch.setenv("XCLIM_B200_NO_TMA", "1")
    b = device.percentile_doy(xd, doy, yidx, L, years, 5, [per], 1 / 3, 1 / 3)
    torch.cuda.synchronize()
    assert torch.equal(torch.nan_to_num(a, nan=-1.0), torch.nan_to_num(b, nan=-1.0))
    exp = O.percentile_doy(x, yidx.astype(np.int64), doy.astype(np.int64), 5, per)[:, 0]
    np.testing.assert_array_equal(a[0].cpu().numpy().reshape((L,) + shape), exp)
