"""The bootstrap launch plan (launch_plan.cuh, through the host build of tests/dispatch_host_build.py) that the GPU
path tests rely on to name the kernel each case runs, pinned on known plans."""
import pytest

from dispatch_host_build import boot_kernel as bootstrap_kernel, boot_plan, exact_years as every_year_exact
from dispatch_host_build import quantile_plan as plan_quantile


@pytest.mark.parametrize("n,w,per,need,kernel", [
    (15, 5, 90.0, 8, "bootstrap5"),
    (16, 5, 90.0, 9, "32x16"),
    (16, 5, 95.0, 5, "bootstrap5"),
    (30, 5, 90.0, 16, "32x16"),      # the WMO 1961-1990 base
    (30, 5, 10.0, 16, "32x16"),
    (30, 5, 99.0, 2, "16x8"),
    (10, 7, 90.0, 8, "16x8"),
    (15, 1, 90.0, 2, "16x8"),
    (40, 5, 90.0, 21, "32x32"),
    (40, 5, 95.0, 11, "32x16"),
    (30, 5, 80.0, 31, None),
    (30, 11, 90.0, 34, None),
    (15, 5, 50.0, 38, None),
])
def test_plan_and_kernel(n, w, per, need, kernel):
    got_need, top = plan_quantile(per, 1 / 3, 1 / 3, n * w)
    assert got_need == need
    assert top == (per >= 50.0)      # the top side wins ties
    assert bootstrap_kernel(n, w, per) == kernel


def test_dispatch_switches():
    assert bootstrap_kernel(15, 5, 90.0, boot_v1=True) == "16x8"
    assert bootstrap_kernel(15, 5, 90.0, year_len=8) == "16x8"       # bootstrap5 needs year_len > 8
    assert bootstrap_kernel(17, 5, 95.0) == "16x8"                   # and at most 16 base years
    assert every_year_exact(33) and not every_year_exact(32)


@pytest.mark.parametrize("n,year_len,C,mask,expect", [
    # the WMO 1961-1990 base: bootstrap_kernel<32, 16>, 6 CTAs per SM, at least 4 W = 20 days per chunk
    (30, 365, 161, False, ("32x16", 20, 19)),
    (30, 365, 161, True, ("32x16", 32, 12)),            # mask words have one writer: chunks of whole words
    (30, 365, 100_000, False, ("32x16", 183, 2)),
    (30, 365, 100_000, True, ("32x16", 192, 2)),
    (30, 360, 30_000, True, ("32x16", 96, 4)),
    (15, 365, 161, True, ("bootstrap5", 32, 12)),       # one warp per CTA, 12 CTAs per SM
    (15, 40, 161, True, ("bootstrap5", 32, 2)),
    (15, 365, 100_000, True, ("bootstrap5", 365, 1)),
])
def test_day_split(n, year_len, C, mask, expect):
    kernel, chunks, per, _ = boot_plan(n, 5, 90.0, year_len=year_len, mask=mask, C=C)
    assert (kernel, per, chunks) == expect
    if mask:
        assert per % 32 == 0 or per == year_len
