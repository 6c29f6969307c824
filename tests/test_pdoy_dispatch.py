"""The percentile_doy launch plan (launch_plan.cuh, through the host build of tests/dispatch_host_build.py) that the
GPU path tests rely on to name the kernels each case runs, pinned on known plans: every template instance, the TMA
eligibility, the shared-memory and selection caps, table mode's day segmentation and the day splits."""
import datetime

import numpy as np
import pytest

from dispatch_host_build import PDOY_INSTANCES as INSTANCES, Unsupported
from dispatch_host_build import pdoy_kernels as kernels, pdoy_plan as kernel_plan, split_plan as split_days
from xb_helpers import uniform_calendar


def _standard(start, end):
    """(doy, year ordinal, n_years) of the daily standard calendar from ``start`` to ``end`` inclusive."""
    from xclim_b200 import TimeAxis
    d0, d1 = (datetime.date.fromisoformat(s) for s in (start, end))
    ta = TimeAxis.daily(start, (d1 - d0).days + 1, "standard")
    years = np.unique(ta.year)
    return ta.doy, np.searchsorted(years, ta.year), len(years)


def _uniform(L, N):
    doy, year = uniform_calendar(L, N)
    return doy, year, N


WMO = ("1961-01-01", "1990-12-31")
MIDYEAR = ("1960-07-01", "1990-06-30")

# (calendar, window, percentiles, layout, kernels); calendar: (L, years) uniform or (start, end) standard;
# layout: keyword arguments of kernel_plan besides C (default C = 141)
CASES = [
    ((365, 6), 5, [90], {}, {"w5p<8, false>"}),
    ((365, 20), 5, [90], {}, {"w5p<16, false>"}),
    ((365, 30), 5, [90], {"C": 140}, {"w5t<14>"}),
    ((365, 30), 5, [10], {"C": 140}, {"w5t<14>"}),
    ((360, 31), 5, [90], {"C": 140}, {"w5t<15>"}),
    ((365, 32), 5, [92], {"C": 140}, {"w5t<16>"}),
    ((360, 32), 5, [8], {"C": 140}, {"w5t<16>"}),
    ((365, 32), 5, [90], {"C": 140}, {"uniform<32, false>"}),     # need 17: no 32-year TMA at per 90
    ((365, 30), 5, [90], {"C": 141, "ldx": 148}, {"w5t<14>"}),    # band view, ldx = 4k > C
    ((365, 30), 5, [90], {"C": 140, "no_tma": True}, {"w5p<16, false>"}),
    ((365, 30), 5, [90], {"C": 141}, {"w5p<16, false>"}),         # ldx % 4 != 0
    ((365, 30), 5, [90], {"C": 140, "ldx": 147}, {"w5p<16, false>"}),
    ((365, 30), 5, [90], {"C": 140, "ldx": 144, "aligned16": False}, {"w5p<16, false>"}),
    ((365, 29), 5, [90], {"C": 140}, {"w5p<16, false>"}),         # TMA needs 30..32 years
    ((365, 33), 5, [95], {"C": 140}, {"w5p<16, false>"}),
    ((365, 30), 3, [95], {}, {"uniform<8, false>"}),
    ((365, 30), 3, [90], {}, {"uniform<16, false>"}),
    ((365, 30), 9, [90], {}, {"uniform<32, false>"}),
    ((365, 16), 13, [90], {}, {"uniform<32, false>"}),            # 198 KB of shared memory
    ((365, 16), 15, [90], {}, {"generic<32>"}),                   # 231 KB: over the cap
    ((365, 30), 1, [90], {}, {"generic<4>"}),
    ((365, 30), 5, [75], {}, {"generic<64>"}),
    ((365, 30), 5, [50], {}, {"select"}),
    ((365, 30), 25, [50], {}, {"select"}),                        # 750 samples
    (WMO, 5, [90, 10], {}, {"w5p<16, true>", "generic<16>"}),
    (WMO, 5, [99], {}, {"w5p<8, true>", "generic<4>"}),
    (WMO, 3, [95], {}, {"uniform<8, true>", "generic<8>"}),
    (WMO, 3, [90], {}, {"uniform<16, true>", "generic<16>"}),
    (WMO, 7, [90], {}, {"uniform<32, true>", "generic<32>"}),
    (MIDYEAR, 5, [90, 10], {}, {"w5p<16, true>", "generic<16>"}),
    (MIDYEAR, 7, [90], {}, {"uniform<32, true>", "generic<32>"}),
    (WMO, 1, [90], {}, {"generic<4>"}),
    ((365, 30), 5, [0, 10, 50, 75, 90, 99, 100], {"C": 140},
     {"w5p<8, false>", "w5t<14>", "select", "generic<64>"}),
    (WMO, 5, [0, 10, 50, 75, 90, 99, 100], {},
     {"w5p<8, true>", "generic<4>", "w5p<16, true>", "generic<16>", "select", "generic<64>"}),
]


def _calendar(cal):
    return _standard(*cal) if isinstance(cal[0], str) else _uniform(*cal)


def _n_doy(cal):
    return 366 if isinstance(cal[0], str) else cal[0]


def _id(case):
    cal, window, pers, layout, _ = case
    name = f"{cal[0]}" if isinstance(cal[0], str) else f"L{cal[0]}x{cal[1]}"
    extra = "".join(f"-{k}{v}" for k, v in layout.items())
    return f"{name}-w{window}-p{'_'.join(f'{p:g}' for p in pers)}{extra}"


@pytest.mark.parametrize("cal,window,pers,layout,expect", CASES, ids=[_id(c) for c in CASES])
def test_dispatch_pins(cal, window, pers, layout, expect):
    doy, year, ny = _calendar(cal)
    kw = dict(layout)
    C = kw.pop("C", 141)
    assert kernels(doy, year, _n_doy(cal), ny, window, pers, C, **kw) == expect


def test_pins_cover_every_instance():
    seen = set()
    for cal, window, pers, layout, _ in CASES:
        doy, year, ny = _calendar(cal)
        kw = dict(layout)
        C = kw.pop("C", 141)
        seen |= kernels(doy, year, _n_doy(cal), ny, window, pers, C, **kw)
    assert seen == set(INSTANCES) and len(INSTANCES) == 19


def test_selection_sample_cap():
    doy, year = uniform_calendar(365, 31)
    with pytest.raises(Unsupported):
        kernel_plan(doy, year, 365, 31, 25, [50.0], 64)            # 775 samples
    with pytest.raises(Unsupported):
        kernel_plan(doy, year, 365, 31, 4, [90.0], 64)             # even window


def test_table_mode_segments():
    """Standard calendar: per-day lists on days 3..363, generic on the edge days; a mid-year start also
    leaves the h days before its first day-of-year and after its last one to the generic kernel, and a fast
    run shorter than 8 days goes there too."""
    def spans(cal, window, per):
        doy, year, ny = _standard(*cal)
        return [(ln.kernel, ln.a, ln.b) for ln in kernel_plan(doy, year, 366, ny, window, [per], 141)]
    assert spans(WMO, 5, 90.0) == [("generic<16>", 0, 2), ("w5p<16, true>", 2, 363), ("generic<16>", 363, 366)]
    # 1960-07-01 is day 183 of a leap year, 1990-06-30 day 181 of a common year
    assert spans(MIDYEAR, 5, 10.0) == [("generic<16>", 0, 2), ("w5p<16, true>", 2, 180), ("generic<16>", 180, 183),
                                       ("w5p<16, true>", 183, 363), ("generic<16>", 363, 366)]
    # 1961-01-10: days 3..7 are a 5-day fast run
    assert spans(("1961-01-10", "1991-01-09"), 5, 99.0) == [
        ("generic<4>", 0, 2), ("generic<4>", 2, 7), ("generic<4>", 7, 11), ("w5p<8, true>", 11, 363),
        ("generic<4>", 363, 366)]
    assert spans(WMO, 7, 90.0) == [("generic<32>", 0, 3), ("uniform<32, true>", 3, 362), ("generic<32>", 362, 366)]


def test_percentile_offsets_in_one_call():
    doy, year = uniform_calendar(365, 30)
    plan = kernel_plan(doy, year, 365, 30, 5, [0, 10, 50, 75, 90, 99, 100], 140)
    assert [(ln.ip, ln.kernel) for ln in plan] == [
        (0, "w5p<8, false>"), (1, "w5t<14>"), (2, "select"), (3, "generic<64>"), (4, "w5t<14>"), (5, "w5p<8, false>"),
        (6, "w5p<8, false>")]


@pytest.mark.parametrize("nd,cblocks,ctas,min_per,pairs,expect", [
    (365, 2, 16, 40, True, (10, 40)),          # the small parity grids: shortest chunks
    (365, 704, 16, 40, True, (3, 122)),        # a few long chunks, the last one odd (121 days)
    (361, 704, 16, 40, True, (3, 122)),
    (365, 528, 12, 72, False, (3, 122)),
    (365, 10_000, 12, 40, True, (1, 365)),
    (366, 2, 8, 1, False, (366, 1)),
])
def test_split_days(nd, cblocks, ctas, min_per, pairs, expect):
    assert split_days(nd, cblocks, ctas, min_per, pairs, sms=132) == expect


@pytest.mark.parametrize("nd,cblocks,ctas,min_per,pairs,align,sms,expect", [
    (365, 2, 12, 20, False, 32, 132, (12, 32)),      # whole mask words: 11 chunks of 32 days and one of 13
    (365, 300, 6, 20, False, 32, 132, (3, 128)),     # 122 days rounded up to four words
    (365, 10_000, 6, 20, False, 32, 132, (1, 365)),  # one chunk: the whole year
    (40, 2, 12, 20, False, 32, 114, (2, 32)),        # the last chunk keeps the remaining 8 days
    (365, 2, 16, 40, True, 32, 132, (6, 64)),        # whole pairs, then whole words
    (30, 2, 6, 4, False, 32, 132, (1, 30)),          # a year shorter than one word: one chunk
])
def test_split_days_aligned(nd, cblocks, ctas, min_per, pairs, align, sms, expect):
    chunks, per = split_days(nd, cblocks, ctas, min_per, pairs, sms=sms, align=align)
    assert (chunks, per) == expect
    assert per == nd or per % align == 0
