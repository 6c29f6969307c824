"""GPU parity of every kernel behind xc_percentile_doy_f32 against the oracle, bit for bit.

The dispatch picks, per percentile, the generic kernel (4..64 kept order statistics), the selection kernel,
the ring kernel (uniform<8|16|32>), the paired window-5 kernel (w5p<8|16>) -- each of the last two on uniform
years or through the (year, day-of-year) table -- or the TMA-fed window-5 kernel (w5t, 30..32 uniform years).
Each case names the kernels it is meant to reach (the launch plan the launcher executes), checks that
name against the launches torch.profiler records, and compares the raw (n_per, n_doy, C) table with the
oracle's table before its 365 -> 366 re-interpolation and with the generic kernel's.  The data hold scattered
NaN, whole NaN years on some days, an all-NaN and a one-value cell, ties, signed zeros, and cells whose
interpolation meets +-inf or overflows float32; the layouts hold partial cell blocks, C % 4 != 0, row
strides above C and a base pointer off 16-byte alignment.
"""
import datetime
import re
import warnings

import numpy as np
import pytest

from dispatch_host_build import Unsupported, pdoy_plan as kernel_plan, quantile_plan as plan_quantile
from oracle import xclim_oracle as O
from xb_helpers import plant_infinite_samples, uniform_calendar

pytestmark = pytest.mark.gpu

A3 = 1 / 3
WMO = ("1961-01-01", "1990-12-31")
MIDYEAR = ("1960-07-01", "1990-06-30")


def _calendar(cal):
    """(doy, year ordinal, n_years, n_doy) of (L, years) uniform years or a (start, end) standard calendar."""
    if isinstance(cal[0], str):
        from xclim_b200 import TimeAxis
        d0, d1 = (datetime.date.fromisoformat(s) for s in cal)
        ta = TimeAxis.daily(cal[0], (d1 - d0).days + 1, "standard")
        years = np.unique(ta.year)
        return ta.doy.astype(np.int64), np.searchsorted(years, ta.year), len(years), 366
    L, n = cal
    doy, year = uniform_calendar(L, n)
    return doy, year, n, L


def _raw_table(x, year, doy, n_doy, window, pers):
    """(n_per, n_doy, C) day-of-year quantiles of O.percentile_doy before its 365 -> 366 re-interpolation"""
    rr = O.rolling_construct_center(x, window)
    ny = int(year.max()) + 1
    rrr = np.full((n_doy, ny * window) + x.shape[1:], np.nan, dtype=rr.dtype)
    for k in range(window):
        rrr[doy - 1, year * window + k] = rr[:, k]
    q = np.stack([O.nan_quantile(rrr[d], np.asarray(pers) / 100.0, A3, A3) for d in range(n_doy)])
    return np.moveaxis(q, 1, 0)


def _hostile(rng, doy, year, C, pers, seed):
    """(T, C) float32 on a 0.25 grid; cell 0 all-NaN, cell 1 one valid value, cell 2 signed zeros, cells
    3 + 7k whole NaN years on some days, five cells per percentile from cell 5 on with infinite samples."""
    T = doy.size
    x = 288 + 12 * np.sin(2 * np.pi * (doy - 110) / 365)[:, None] + 3 * rng.standard_normal((T, C))
    x = (np.round(x * 4) / 4).astype(np.float32)
    x[rng.random(x.shape) < 0.01] = np.nan
    gap = ((year % 4 == 1) & (doy % 9 < 3))[:, None] & (np.arange(C) % 7 == 3)[None, :]
    x[gap] = np.nan
    x[:, 0] = np.nan
    x[:, 1] = np.nan
    x[T // 3, 1] = 7.0
    x[:, 2] = np.where(rng.random(T) < 0.5, np.float32(0.0), np.float32(-0.0))
    x[rng.random(T) < 0.1, 2] = 0.25
    qs = sorted({p / 100.0 for p in pers})
    plant_infinite_samples(x, qs, range(5, 5 + 5 * len(qs)), seed=seed)
    return x


def _place(x, layout, cuda):
    """Device (T, C) view of x: "plain" contiguous, "band" rows of 4k > C floats, "odd" an odd row stride,
    "shift" a base pointer 4 bytes past 16-byte alignment.  Floats outside the view are +-1e9."""
    import torch
    T, C = x.shape
    xh = torch.from_numpy(x)
    if layout == "plain":
        return xh.to(cuda)
    ldx, c0 = {"band": ((C + 3) // 4 * 4 + 4, 4), "odd": ((C + 8) | 1, 3), "shift": ((C + 3) // 4 * 4 + 8, 1)}[layout]
    wide = torch.full((T, ldx), 1e9, dtype=torch.float32)
    wide[:, ::2] = -1e9
    wide[:, c0:c0 + C] = xh
    xd = wide.to(cuda)[:, c0:c0 + C]
    assert xd.stride(0) == ldx
    return xd


_INST = re.compile(r"percentile_doy_(\w+?)_kernel(?:<([^>]*)>|I((?:L[bi]\d+E)+)E)?")


def _instances(names):
    """template instances ("w5p<16, true>", "select", ...) among demangled or mangled kernel names"""
    out = set()
    for name in names:
        m = _INST.search(name)
        if not m:
            continue
        base, dem, man = m.groups()
        args = dem or (", ".join({"b1": "true", "b0": "false"}.get(a, a[1:]) for a in re.findall(r"L([bi]\d+)E", man))
                       if man else None)
        out.add(f"{base}<{args}>" if args else base)
    return out


def _profiled(fn):
    """fn()'s result and the percentile_doy instances it launched (None when the profiler saw no kernel)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    kernels = [n for n in names if "kernel" in n.lower() or n.startswith("_Z")]
    return out, (_instances(kernels) if kernels else None)


def _check(xd, x_host, cal, window, pers, expect, sel=None, no_tma=False):
    """Launches the plan names, the profiler's witness, the oracle's bits and the generic kernel's."""
    import torch
    from xclim_b200 import device
    doy, year, ny, n_doy = _calendar(cal)
    C = xd.shape[1]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    plan = kernel_plan(doy, year, n_doy, ny, window, pers, C, ldx=xd.stride(0), aligned16=xd.data_ptr() % 16 == 0,
                       no_tma=no_tma, sms=sms)
    assert {ln.kernel for ln in plan} == expect
    got, seen = _profiled(lambda: device.percentile_doy(xd, doy, year, n_doy, ny, window, pers, A3, A3))
    if seen is None:
        warnings.warn("torch.profiler recorded no kernels: the launched instances are not witnessed")
    else:
        assert seen == expect
    cols = slice(None) if sel is None else torch.from_numpy(sel).to(xd.device)
    exp = _raw_table(x_host, year, doy, n_doy, window, pers)
    np.testing.assert_array_equal(got[:, :, cols].cpu().numpy(), exp)
    # the generic kernel holds at most 64 order statistics: the selection kernel's percentiles have no twin
    for ip, per in enumerate(pers):
        if plan_quantile(per, A3, A3, ny * window)[0] <= 64:
            gen = device.percentile_doy(xd, doy, year, n_doy, ny, window, [per], A3, A3, force_generic=True)
            np.testing.assert_array_equal(gen[0].cpu().numpy(), got[ip].cpu().numpy())
    return plan


CASES = [
    # calendar, window, percentiles, C, layout, kernels
    ((365, 6), 5, [90.0], 141, "plain", {"w5p<8, false>"}),
    ((365, 20), 5, [90.0], 140, "odd", {"w5p<16, false>"}),
    ((365, 30), 3, [95.0], 141, "plain", {"uniform<8, false>"}),
    ((365, 30), 3, [90.0], 141, "band", {"uniform<16, false>"}),
    ((365, 30), 9, [90.0], 140, "odd", {"uniform<32, false>"}),
    ((365, 16), 13, [90.0], 141, "plain", {"uniform<32, false>"}),     # 198 KB of shared memory: under the cap
    ((365, 16), 15, [90.0], 141, "plain", {"generic<32>"}),            # 231 KB: over it
    ((360, 30), 1, [90.0], 141, "shift", {"generic<4>"}),
    ((365, 30), 5, [75.0], 141, "plain", {"generic<64>"}),             # need 38
    ((365, 30), 5, [50.0], 141, "odd", {"select"}),
    ((365, 30), 25, [50.0], 141, "plain", {"select"}),                 # 750 samples, the cap is 768
    ((365, 30), 5, [0.0, 10.0, 50.0, 75.0, 90.0, 99.0, 100.0], 140, "plain",
     {"w5p<8, false>", "w5t<14>", "select", "generic<64>"}),
    (WMO, 5, [90.0, 10.0], 141, "plain", {"w5p<16, true>", "generic<16>"}),
    (WMO, 5, [99.0], 141, "odd", {"w5p<8, true>", "generic<4>"}),
    (WMO, 3, [95.0], 141, "plain", {"uniform<8, true>", "generic<8>"}),
    (WMO, 3, [90.0], 141, "band", {"uniform<16, true>", "generic<16>"}),
    (WMO, 7, [90.0], 141, "plain", {"uniform<32, true>", "generic<32>"}),
    (WMO, 5, [0.0, 10.0, 50.0, 75.0, 90.0, 99.0, 100.0], 141, "plain",
     {"w5p<8, true>", "generic<4>", "w5p<16, true>", "generic<16>", "select", "generic<64>"}),
    (MIDYEAR, 5, [90.0, 10.0], 141, "plain", {"w5p<16, true>", "generic<16>"}),
    (MIDYEAR, 5, [99.0], 141, "shift", {"w5p<8, true>", "generic<4>"}),
    (MIDYEAR, 3, [95.0], 141, "plain", {"uniform<8, true>", "generic<8>"}),
    (MIDYEAR, 3, [90.0], 141, "odd", {"uniform<16, true>", "generic<16>"}),
    (MIDYEAR, 7, [90.0], 141, "plain", {"uniform<32, true>", "generic<32>"}),
    (("1961-01-10", "1991-01-09"), 5, [99.0], 141, "plain", {"w5p<8, true>", "generic<4>"}),   # a 5-day fast run
]


def _case_id(c):
    cal, window, pers, C, layout, _ = c
    name = cal[0] if isinstance(cal[0], str) else f"L{cal[0]}x{cal[1]}"
    return f"{name}-w{window}-p{'_'.join(f'{p:g}' for p in pers)}-C{C}-{layout}"


@pytest.mark.parametrize("cal,window,pers,C,layout,expect", CASES, ids=[_case_id(c) for c in CASES])
def test_percentile_doy_paths(cuda, monkeypatch, cal, window, pers, C, layout, expect):
    monkeypatch.delenv("XCLIM_B200_NO_TMA", raising=False)
    doy, year, _, _ = _calendar(cal)
    rng = np.random.default_rng(500 + window + int(sum(pers)) + len(doy))
    x = _hostile(rng, doy, year, C, pers, seed=window)
    _check(_place(x, layout, cuda), x, cal, window, pers, expect)


@pytest.mark.parametrize("L", [365, 360])
@pytest.mark.parametrize("years,per,C,layout", [
    (30, 90.0, 140, "plain"), (31, 90.0, 140, "plain"), (32, 92.0, 140, "plain"),
    (30, 10.0, 141, "band"), (31, 90.0, 141, "band"), (32, 8.0, 141, "band"),
])
def test_percentile_doy_tma_kernels(cuda, monkeypatch, L, years, per, C, layout):
    """w5t<N - 16> for N = 30..32 years (also on a band view of rows of 4k > C floats) and, with
    XCLIM_B200_NO_TMA, the lane-by-lane w5p<16> with its cp.async staging on the same data."""
    rng = np.random.default_rng(700 + years + L)
    doy, year = uniform_calendar(L, years)
    x = _hostile(rng, doy, year, C, [per], seed=years)
    xd = _place(x, layout, cuda)
    monkeypatch.delenv("XCLIM_B200_NO_TMA", raising=False)
    _check(xd, x, (L, years), 5, [per], {f"w5t<{years - 16}>"})
    monkeypatch.setenv("XCLIM_B200_NO_TMA", "1")
    _check(xd, x, (L, years), 5, [per], {"w5p<16, false>"}, no_tma=True)


def test_percentile_doy_tma_misaligned_base(cuda, monkeypatch):
    """A base pointer 4 bytes past 16-byte alignment (rows of 4k floats) leaves the TMA kernel for w5p<16>."""
    monkeypatch.delenv("XCLIM_B200_NO_TMA", raising=False)
    rng = np.random.default_rng(731)
    doy, year = uniform_calendar(365, 30)
    x = _hostile(rng, doy, year, 140, [90.0], seed=31)
    xd = _place(x, "shift", cuda)
    assert xd.stride(0) % 4 == 0 and xd.data_ptr() % 16 == 4
    _check(xd, x, (365, 30), 5, [90.0], {"w5p<16, false>"})


def test_percentile_doy_selection_cap(cuda):
    """775 samples per cell (31 years x window 25) are more than the selection kernel holds."""
    import torch
    from xclim_b200 import device
    doy, year = uniform_calendar(365, 31)
    with pytest.raises(Unsupported):
        kernel_plan(doy, year, 365, 31, 25, [50.0], 64)
    x = torch.zeros((365 * 31, 64), dtype=torch.float32, device=cuda)
    with pytest.raises(NotImplementedError, match="768"):
        device.percentile_doy(x, doy, year, 365, 31, 25, [50.0], A3, A3)


# Long day chunks: enough cell blocks that split_days gives each CTA a third of the year (the parity grids
# above get the shortest chunks).  (calendar, window, per, XCLIM_B200_NO_TMA, CTAs per SM of the launch, kernel)
LONG = {
    "w5p": ((365, 30), 5, 90.0, True, 16, "w5p<16, false>"),
    "uniform": ((365, 30), 9, 90.0, False, 12, "uniform<32, false>"),
    "tma": ((365, 30), 5, 10.0, False, 12, "w5t<14>"),
    "table": (WMO, 5, 90.0, False, 16, "w5p<16, true>"),
}


@pytest.mark.parametrize("family", list(LONG))
def test_percentile_doy_long_day_chunks(cuda, monkeypatch, family):
    import torch
    from xclim_b200 import device
    cal, window, per, no_tma, ctas, kernel = LONG[family]
    free, _ = torch.cuda.mem_get_info()
    if free < 16 << 30:
        pytest.skip("needs 16 GB of free HBM")
    if no_tma:
        monkeypatch.setenv("XCLIM_B200_NO_TMA", "1")
    else:
        monkeypatch.delenv("XCLIM_B200_NO_TMA", raising=False)
    doy, year, ny, n_doy = _calendar(cal)
    T = doy.size
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cblocks = (sms * ctas + 2) // 3 + 1            # three chunks of the day range
    C = cblocks * 128 - 4                          # a partial last block; C % 4 == 0 keeps the TMA kernel
    x = device.synth(T, C, kind=1, seed=17)
    rng = np.random.default_rng(19)
    sel = np.unique(np.concatenate([rng.choice(C, 420, replace=False), np.arange(64), [127, 128, 129],
                                    np.arange(C - 40, C)]))
    # hostile data in 40 of the sampled cells, the last one among them
    hot = np.concatenate([sel[:39], [C - 1]])
    xh = _hostile(rng, doy, year, hot.size, [per], seed=23)
    x[:, torch.from_numpy(hot).to(cuda)] = torch.from_numpy(xh).to(cuda)
    xs = x[:, torch.from_numpy(sel).to(cuda)].cpu().numpy()
    expect = {kernel} if family != "table" else {kernel, "generic<16>"}
    plan = _check(x, xs, cal, window, [per], expect, sel=sel, no_tma=no_tma)
    main = next(ln for ln in plan if ln.kernel == kernel)
    assert main.chunks >= 3 and main.per >= 100 and main.last_chunk % 2 == 1, main
    del x
    torch.cuda.empty_cache()
