"""GPU parity of every kernel behind xc_bootstrap_doy_count_f32 against the literal CPU restatement.

The dispatch picks bootstrap5_kernel (window 5, <= 16 base years, <= 8 kept order statistics) or
bootstrap_kernel<KA, KB> with 16x8, 32x16 or 32x32 kept values; above 32 base years every year takes the
exact per-(y, s) loop.  Each case names the kernel it is meant to reach (the launch plan the launcher
executes) and runs on short synthetic years (L = 40 days, so a tenth of the days are year-edge days and
a day chunk ends inside the year) of hostile data: values on a 0.5 grid (ties, x equal to the threshold),
signed zeros, NaN on edge days and whole NaN years, samples with fewer than two values, an all-NaN and a
constant cell, +-inf at the interpolated ranks and finite +-3e38 whose neighbour difference overflows
float32.  Every count is compared bit for bit.
"""
import numpy as np
import pytest

from dispatch_host_build import boot_kernel as bootstrap_kernel, exact_years as every_year_exact
from oracle import xclim_oracle as O

pytestmark = pytest.mark.gpu

L = 40
BIG = np.float32(3e38)


def _hostile(rng, n_years, C, q):
    """(n_years * L, C) float32; cell c gets the pattern c % 10 (cells 0 and 1: all-NaN and constant)."""
    T = n_years * L
    x = (np.round(rng.standard_normal((T, C)) * 6) / 2).astype(np.float32)
    day = np.arange(T) % L
    grp = np.arange(C) % 10
    u = rng.random((T, C))
    edge = ((day < 3) | (day >= L - 3))[:, None]

    def put(g, mask, val):
        m = mask & (grp == g)[None, :]
        x[m] = val if np.ndim(val) == 0 else val[m]

    put(1, x == 0, np.where(u < 0.5, np.float32(0.0), np.float32(-0.0)).astype(np.float32))   # signed zeros
    put(2, edge & (u < 0.3), np.nan)                                      # NaN on year-edge days
    yr = np.arange(T) // L
    put(2, ((yr % 3 == 1) & (day % 7 < 3))[:, None], np.nan)               # whole NaN years at some days
    put(3, u < 0.985, np.nan)                                             # samples of 0, 1, 2 ... values
    put(4, u < 1.3 * (1 - q), np.inf)                                     # +inf reaching the upper ranks
    put(5, u < 1.1 * q, -np.inf)                                          # -inf reaching the lower ranks
    put(6, u < 0.6 * (1 - q), np.inf)                                     # both infinities at both ends
    put(6, u > 1 - 0.6 * q, -np.inf)
    put(7, u < 1.2 * (1 - q), BIG)                                        # finite spans that overflow
    put(7, u > 1 - 0.9 * q, -BIG)
    put(8, u < 0.8 * (1 - q), np.inf)                                     # +inf next to -3e38 and vice versa
    put(8, u > 1 - 0.8 * q, -BIG)
    put(8, (u > 0.5) & (u < 0.5 + 0.3 * (1 - q)), BIG)
    put(9, (u < 0.04) | edge & (u < 0.1), np.nan)
    x[:, 0] = np.nan
    if C > 1:
        x[:, 1] = 1.5
    return x


def _periods(N, monthly):
    """step -> period index for the base years; monthly: four 10-day periods per year."""
    per_year = 4 if monthly else 1
    sp = (np.arange(N * L) // (L // per_year)).astype(np.int32)
    return sp, per_year


def _device(xd, base_start, N, W, per, alpha, beta, op, monthly):
    from xclim_b200 import _lib, device
    sp, ppy = _periods(N, monthly)
    return device.bootstrap_doy_count(xd, base_start, N, L, sp, N * ppy, W, per, alpha, beta, _lib.OPS[op])


def _oracle(x, pre, N, W, per, alpha, beta, op, monthly):
    """in-base periods of O.bootstrap_doy_count on year = block index, doy = 1..L"""
    T = x.shape[0]
    ny = T // L
    year = np.arange(T) // L
    doy = np.arange(T) % L + 1
    ppy = 4 if monthly else 1
    poff = np.arange(ny * ppy + 1) * (L // ppy)
    out = O.bootstrap_doy_count(x, year, doy, poff, (pre, pre + N - 1), window=W, per=per, alpha=alpha, beta=beta,
                                op=op)
    return out[pre * ppy:(pre + N) * ppy]


A3 = (1 / 3, 1 / 3)
CASES = [
    # N, W, per, op, (alpha, beta), kernel, layout
    (15, 5, 90.0, ">", A3, "bootstrap5", "plain"),
    (16, 5, 95.0, ">=", (1.0, 1.0), "bootstrap5", "slice"),
    (2, 5, 90.0, ">", A3, "bootstrap5", "offset"),
    (3, 5, 10.0, "<", A3, "bootstrap5", "monthly"),
    (15, 5, 10.0, "<=", (0.0, 1.0), "bootstrap5", "offset"),
    (16, 5, 90.0, ">", A3, "32x16", "slice"),
    (30, 5, 90.0, ">", A3, "32x16", "plain"),            # the WMO 1961-1990 base
    (30, 5, 10.0, "<", A3, "32x16", "slice"),
    (30, 5, 99.0, ">=", A3, "16x8", "offset"),
    (10, 7, 90.0, "<=", (0.0, 1.0), "16x8", "plain"),
    (15, 1, 90.0, ">", A3, "16x8", "monthly"),
    (16, 3, 10.0, "<", (0.0, 1.0), "16x8", "monthly"),
    (3, 3, 10.0, ">=", (1.0, 1.0), "16x8", "plain"),
    (40, 5, 90.0, ">", A3, "32x32", "plain"),            # N > 32: every year exact
    (33, 5, 95.0, "<", (1.0, 1.0), "32x16", "slice"),
]


@pytest.mark.parametrize("N,W,per,op,ab,kernel,layout", CASES,
                         ids=[f"N{c[0]}-W{c[1]}-p{c[2]:g}-{c[5]}-{c[6]}" for c in CASES])
def test_bootstrap_kernel_paths(cuda, monkeypatch, N, W, per, op, ab, kernel, layout):
    import torch
    alpha, beta = ab
    assert bootstrap_kernel(N, W, per, alpha, beta, year_len=L) == kernel
    rng = np.random.default_rng(1000 + 37 * N + W + int(per))
    C = 161                                               # not a multiple of 32; two CTAs of 128 lanes
    pre = 1 if layout == "offset" else 0
    x = _hostile(rng, pre + N + 1, C, per / 100.0)
    if layout == "slice":                                 # a column slice of a wider tensor: ldx > C
        wide = torch.full((x.shape[0], C + 19), 7.0, dtype=torch.float32, device=cuda)
        wide[:, 5:5 + C] = torch.from_numpy(x).to(cuda)
        xd = wide[:, 5:5 + C]
        assert xd.stride(0) > C
    else:
        xd = torch.from_numpy(x).to(cuda)
    monthly = layout == "monthly"
    monkeypatch.delenv("XCLIM_B200_BOOT_V1", raising=False)
    got = _device(xd, pre * L, N, W, per, alpha, beta, op, monthly).cpu().numpy()
    exp = _oracle(x, pre, N, W, per, alpha, beta, op, monthly)
    np.testing.assert_array_equal(got, exp)
    if kernel == "bootstrap5":                            # the general kernel gives the same bits
        monkeypatch.setenv("XCLIM_B200_BOOT_V1", "1")
        assert bootstrap_kernel(N, W, per, alpha, beta, year_len=L, boot_v1=True) == "16x8"
        v1 = _device(xd, pre * L, N, W, per, alpha, beta, op, monthly).cpu().numpy()
        np.testing.assert_array_equal(v1, got)
    if every_year_exact(N):
        assert kernel in ("32x16", "32x32")


@pytest.mark.parametrize("N,W,per,ok", [(30, 5, 80.0, False), (30, 11, 90.0, False), (30, 5, 90.0, True)])
def test_bootstrap_unsupported_boundary(cuda, N, W, per, ok):
    import torch
    assert (bootstrap_kernel(N, W, per, year_len=L) is not None) == ok
    x = torch.zeros(((N + 1) * L, 8), dtype=torch.float32, device=cuda)
    if ok:
        out = _device(x, 0, N, W, per, 1 / 3, 1 / 3, ">", False)
        assert out.shape == (N, 8) and bool((out == 0).all())
    else:
        with pytest.raises(NotImplementedError):
            _device(x, 0, N, W, per, 1 / 3, 1 / 3, ">", False)


@pytest.mark.parametrize("N,per,op,kernel,lanes,sm_mult", [
    (15, 90.0, ">", "bootstrap5", 32, 12),
    (16, 10.0, "<=", "32x16", 128, 6),
])
def test_bootstrap_single_day_chunk(cuda, monkeypatch, N, per, op, kernel, lanes, sm_mult):
    """Enough cells that the launch keeps the whole year in one day chunk; the same data split into narrow
    column slices (many chunks) must give the same bits, and sampled cells (the last included) the oracle's."""
    import torch
    assert bootstrap_kernel(N, 5, per, year_len=L) == kernel
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    C = sm_mult * sms * lanes + 21
    rng = np.random.default_rng(77 + N)
    x = _hostile(rng, N + 1, C, per / 100.0)
    xd = torch.from_numpy(x).to(cuda)
    monkeypatch.delenv("XCLIM_B200_BOOT_V1", raising=False)
    got = _device(xd, 0, N, 5, per, 1 / 3, 1 / 3, op, False)
    step = 3000
    for c0 in range(0, C, step):
        part = _device(xd[:, c0:c0 + step], 0, N, 5, per, 1 / 3, 1 / 3, op, False)
        assert torch.equal(part, got[:, c0:c0 + step])
    if kernel == "bootstrap5":
        monkeypatch.setenv("XCLIM_B200_BOOT_V1", "1")
        assert torch.equal(_device(xd, 0, N, 5, per, 1 / 3, 1 / 3, op, False), got)
    sel = np.unique(np.concatenate([np.arange(12), rng.choice(C, 51, replace=False), [C - 1]]))
    exp = _oracle(x[:, sel], 0, N, 5, per, 1 / 3, 1 / 3, op, False)
    np.testing.assert_array_equal(got[:, sel].cpu().numpy(), exp)


def _boot_years_composed(x, N, Lc, years, window, per, op):
    """O.bootstrap_doy_count restricted to the periods of base years ``years`` (first N blocks of Lc
    steps are the base): the table of every altered base series is computed once and serves both the
    yearly and the monthly sums.  Returns {y: (Lc, C) float64 mean exceedance per step}."""
    xb = x[:N * Lc]
    yb = np.arange(N * Lc) // Lc
    db = np.arange(N * Lc) % Lc + 1
    out = {}
    for y in years:
        acc = []
        blk = x[y * Lc:(y + 1) * Lc]
        for s in range(N):
            if s == y:
                continue
            z = xb.copy()
            z[y * Lc:(y + 1) * Lc] = xb[s * Lc:(s + 1) * Lc]
            tab = O.percentile_doy(z, yb, db, window, per)[:, 0]
            acc.append(O.compare(blk, op, tab).astype(np.int64))
        out[y] = np.sum(acc, axis=0)
    return out


@pytest.mark.parametrize("calendar", ["noleap", "360_day"])
def test_tx90p_bootstrap_30_year_base(cuda, calendar):
    """indices.tx90p(bootstrap=True) on a 1961-1990 base (bootstrap_kernel<32, 16>), YS and MS, a few cells:
    every period of three base years against the oracle's composition, out-of-base years against the plain
    index."""
    from xclim_b200 import calendar as xcal, indices
    from xb_helpers import make_field
    Lc = 365 if calendar == "noleap" else 360
    assert bootstrap_kernel(30, 5, 90.0, year_len=Lc) == "32x16"
    rng = np.random.default_rng(61 + Lc)
    nyears = 32
    t = np.arange(nyears * Lc)
    x = 288 + 12 * np.sin(2 * np.pi * (t % Lc - 110) / Lc)[:, None] + 3 * rng.standard_normal((t.size, 3))
    x = (np.round(x * 2) / 2).astype(np.float32)
    x[rng.random(x.shape) < 0.003] = np.nan
    da = make_field(x, "1961-01-01", calendar=calendar, units="K")
    base = da.isel_time(da.time.sel_years(1961, 1990))
    pdoy = xcal.select_percentile(xcal.percentile_doy(base, window=5, per=90.0), 90.0)
    years = (0, 17, 29)
    sums = _boot_years_composed(x, 30, Lc, years, 5, 90.0, ">")
    for freq in ("YS", "MS"):
        got = indices.tx90p(da, pdoy, freq=freq, bootstrap=True).values
        poff = np.asarray(da.time.period_offsets(freq))
        labels = da.time.period_labels(freq)
        yrs = np.array([int(s[:4]) for s in labels])
        for y in years:
            for p in np.nonzero(yrs == 1961 + y)[0]:
                a, b = poff[p] - y * Lc, poff[p + 1] - y * Lc
                np.testing.assert_array_equal(got[p], sums[y][a:b].sum(axis=0) / 29.0)
        plain = indices.tx90p(da, pdoy, freq=freq).values.astype(np.float64)
        np.testing.assert_array_equal(got[yrs > 1990], plain[yrs > 1990])
