"""GPU parity of xc_bootstrap_doy_index_f32 (the MASK mode of the bootstrap kernels + bootstrap_reduce_kernel) and of
the bootstrap=True paths of the spell and precipitation indices.

- On every dispatch path, with the hostile L = 40 data of test_gpu_bootstrap_paths.py, the days-over reducer with no
  floor gives the count kernel's results bit for bit (the popcount of the masks equals the counts).
- On small cases the mask words equal the oracle's per-(y, s) exceedance bits, with and without a floor.
- Spell, count and fraction results equal the oracle-backed restatement of the C-ABI contract
  (tests/fake_bootstrap.py) bit for bit, and the public indices equal the literal oracle on three calendars.
"""
import numpy as np
import pytest

import fake_bootstrap
import test_gpu_bootstrap_paths as paths
from fake_device import OP_NAME
from oracle import bootstrap_oracle as B
from oracle import xclim_oracle as O
from test_bootstrap_index_cpu import label_years
from xb_helpers import make_field

pytestmark = pytest.mark.gpu
L = paths.L


def _index(xd, pre, N, W, per, ab, op, monthly, kind, **kw):
    from xclim_b200 import _lib, device
    sp, ppy = paths._periods(N, monthly)
    return device.bootstrap_doy_index(xd, pre * L, N, L, sp, N * ppy, W, per, ab[0], ab[1], _lib.OPS[op], kind, **kw)


def _bits(scratch, N, C):
    """(pair, day, cell) 0/1 of the masks left in the scratch (one tile): bit d % 32 of word d // 32."""
    Wd = (L + 31) // 32
    m = scratch[:N * (N - 1) * Wd * C * 4].cpu().numpy().view(np.uint32).reshape(N * (N - 1), Wd, 1, C)
    b = (m >> np.arange(32, dtype=np.uint32)[None, None, :, None]) & 1
    return b.reshape(N * (N - 1), Wd * 32, C)[:, :L]


@pytest.mark.parametrize("N,W,per,op,ab,kernel,layout", paths.CASES,
                         ids=[f"N{c[0]}-W{c[1]}-p{c[2]:g}-{c[5]}-{c[6]}" for c in paths.CASES])
def test_mask_popcount_equals_counts(cuda, monkeypatch, N, W, per, op, ab, kernel, layout):
    import torch
    from dispatch_host_build import boot_plan
    assert boot_plan(N, W, per, ab[0], ab[1], year_len=L, mask=True)[0] == kernel
    rng = np.random.default_rng(2000 + 37 * N + W + int(per))
    C = 161
    pre = 1 if layout == "offset" else 0
    x = paths._hostile(rng, pre + N + 1, C, per / 100.0)
    if layout == "slice":
        wide = torch.full((x.shape[0], C + 19), 7.0, dtype=torch.float32, device=cuda)
        wide[:, 5:5 + C] = torch.from_numpy(x).to(cuda)
        xd = wide[:, 5:5 + C]
    else:
        xd = torch.from_numpy(x).to(cuda)
    monthly = layout == "monthly"
    monkeypatch.delenv("XCLIM_B200_BOOT_V1", raising=False)
    cnt = paths._device(xd, pre * L, N, W, per, ab[0], ab[1], op, monthly).cpu().numpy()
    got, scratch = _index(xd, pre, N, W, per, ab, op, monthly, "count")
    np.testing.assert_array_equal(got.cpu().numpy(), cnt)
    # the masks themselves: bits per (y, s) summed over s and days == N - 1 times the mean
    bits = _bits(scratch, N, C)
    sp, ppy = paths._periods(N, monthly)
    tot = np.zeros((N * ppy, C))
    for y in range(N):
        yb = bits[y * (N - 1):(y + 1) * (N - 1)].sum(0)
        for p in np.unique(sp[y * L:(y + 1) * L]):
            tot[p] += yb[sp[y * L:(y + 1) * L] == p].sum(0)
    np.testing.assert_array_equal(tot / (N - 1), cnt)


@pytest.mark.parametrize("N,W,per,op,floor", [(3, 5, 90.0, ">", None), (4, 3, 75.0, ">=", 0.5), (3, 5, 10.0, "<", None),
                                              (4, 5, 95.0, ">", 2.0)])
def test_mask_bits_equal_oracle(cuda, N, W, per, op, floor):
    import torch
    rng = np.random.default_rng(7 + N + W)
    C = 40
    x = paths._hostile(rng, N, C, per / 100.0)
    got, scratch = _index(torch.from_numpy(x).to(cuda), 0, N, W, per, paths.A3, op, False, "count", floor=floor)
    bits = _bits(scratch, N, C).astype(bool)
    year = np.repeat(np.arange(N), L)
    doy = np.tile(np.arange(1, L + 1), N)
    for y in range(N):
        for s in range(N):
            if s == y:
                continue
            z = x.copy()
            z[year == y] = x[year == s]
            tab = O.percentile_doy(z, year, doy, W, per, *paths.A3)[:, 0]
            if floor is not None:
                with np.errstate(invalid="ignore"):
                    tab = np.where(tab > floor, tab, floor)
            exp = O.compare(x[year == y], op, tab)
            pair = y * (N - 1) + (s if s < y else s - 1)
            np.testing.assert_array_equal(bits[pair], exp, err_msg=f"y={y} s={s}")


CASES = [("spell", 1, True), ("spell", 3, True), ("spell", 3, False), ("spell", 6, False), ("spell", 6, True),
         ("count", 1, True), ("sum", 1, True)]


@pytest.mark.parametrize("kind,rw,rbrl", CASES)
@pytest.mark.parametrize("N,W,per,op", [(4, 5, 80.0, ">"), (3, 3, 20.0, "<"), (5, 5, 90.0, ">=")])
def test_index_equals_oracle(cuda, kind, rw, rbrl, N, W, per, op):
    import torch
    from xclim_b200 import _lib
    if kind != "spell" and op not in (">", ">="):
        pytest.skip("the precipitation indices take > / >=")
    rng = np.random.default_rng(11 + N)
    C = 70
    x = paths._hostile(rng, N + 1, C, per / 100.0)
    x[:, 10:30] = np.abs(np.round(rng.gamma(0.7, 3.0, (x.shape[0], 20)) * 2) / 2) * (rng.random((x.shape[0], 20)) < .6)
    xd = torch.from_numpy(x).to(cuda)
    sp, ppy = paths._periods(N, True)
    P = N * ppy
    floor = 1.0 if kind != "spell" else None
    wet = None
    if kind == "sum":
        xb = x[:N * L]
        tot = np.where(O.compare(xb, op, 1.0), xb, np.float32(0))
        wet = torch.from_numpy(np.stack([tot[a:a + L // ppy].sum(0, dtype=np.float64)
                                         for a in range(0, N * L, L // ppy)]).astype(np.float32)).to(cuda)
    kw = dict(run_window=rw, resample_before_rl=rbrl, floor=floor, wet_total=wet)
    got, _ = _index(xd, 0, N, W, per, paths.A3, op, True, kind, **kw)
    exp, _ = fake_bootstrap.bootstrap_doy_index(torch.from_numpy(x), 0, N, L, sp, P, W, per, *paths.A3, _lib.OPS[op],
                                                kind, **{**kw, "wet_total": None if wet is None else wet.cpu()})
    assert OP_NAME[_lib.OPS[op]] == op
    np.testing.assert_array_equal(got.cpu().numpy(), exp.numpy())


@pytest.mark.parametrize("C", [1, 127, 129, 1409, 4100])
def test_cell_tiles(cuda, C):
    """A scratch that forces several tiles (ragged last one) and ldx > C views give the one-tile bits."""
    import torch
    from xclim_b200 import _lib
    N = 4
    rng = np.random.default_rng(C)
    x = paths._hostile(rng, N, C + 3, 0.9)
    wide = torch.from_numpy(x).to(cuda)
    xd = wide[:, 2:2 + C]
    sp, ppy = paths._periods(N, True)
    one, _ = _index(xd, 0, N, 5, 90.0, paths.A3, ">", True, "spell", run_window=3, resample_before_rl=False)
    per_cell = int(_lib.load().xc_bootstrap_doy_index_scratch_bytes(N, L, 1))
    if C > 128:
        tiles, _ = _index(xd, 0, N, 5, 90.0, paths.A3, ">", True, "spell", run_window=3, resample_before_rl=False,
                          scratch_bytes=per_cell * 128 * max(1, C // 384))
        np.testing.assert_array_equal(tiles.cpu().numpy(), one.cpu().numpy())
    ref, _ = _index(xd.contiguous(), 0, N, 5, 90.0, paths.A3, ">", True, "spell", run_window=3,
                    resample_before_rl=False)
    np.testing.assert_array_equal(one.cpu().numpy(), ref.cpu().numpy())
    with pytest.raises(Exception, match="scratch"):
        _index(xd, 0, N, 5, 90.0, paths.A3, ">", True, "spell", run_window=3, scratch_bytes=per_cell * min(C, 128) - 4)


def _series(calendar, years, cells, seed, kind):
    rng = np.random.default_rng(seed)
    n = {"noleap": 365, "360_day": 360}.get(calendar)
    T = n * len(years) if n else int(sum(366 if y % 4 == 0 else 365 for y in years))
    t = np.arange(T)
    if kind == "tas":
        x = 288 + 8 * np.sin(2 * np.pi * t / 365.25)[:, None] + 3 * rng.standard_normal((T, cells))
        x += 2.5 * np.repeat(rng.standard_normal((T // 4 + 1, cells)), 4, axis=0)[:T]
    else:
        x = rng.gamma(0.6, 5.0, (T, cells)) * (rng.random((T, cells)) < 0.5)
    x = x.astype(np.float32)
    return x, make_field(x, f"{years[0]}-01-01", calendar=calendar, units="K" if kind == "tas" else "mm/d")


@pytest.mark.parametrize("calendar", ["noleap", "360_day", "standard"])
@pytest.mark.parametrize("freq", ["YS", "MS", "QS-DEC", "YS-JUL"])
def test_public_indices_equal_oracle(cuda, calendar, freq):
    from xclim_b200 import calendar as xcal, indices
    years = list(range(2003, 2008))
    cmd = {"standard": 366, "noleap": 365, "360_day": 360}[calendar]
    t_x, tas = _series(calendar, years, 3, 1, "tas")
    p_x, pr = _series(calendar, years, 3, 2, "pr")
    feb29 = (np.asarray(tas.time.month) == 2) & (np.asarray(tas.time.day) == 29)

    def oracle(da, x, index, per, fraction=False):
        t = da.time
        return B.bootstrap_doy_index(x, t.year, t.doy, t.bootstrap_group_ids(freq), label_years(da, freq),
                                     t.period_offsets(freq), (2004, 2006), index, window=5, per=per, feb29=feb29,
                                     fraction=fraction)

    def pdoy(da, per):
        base = da.isel_time(da.time.sel_years(2004, 2006))
        return xcal.select_percentile(xcal.percentile_doy(base, window=5, per=per), per)
    for rbrl, w in ((True, 6), (False, 3)):
        got = indices.warm_spell_duration_index(tas, pdoy(tas, 80.0), window=w, freq=freq, resample_before_rl=rbrl,
                                                bootstrap=True)
        exp = oracle(tas, t_x, B.spell_index("warm_spell_duration_index", w, rbrl, cal_max_doy=cmd), 80.0)
        np.testing.assert_array_equal(got.values, exp, err_msg=f"wsdi {rbrl}")
    got = indices.cold_spell_duration_index(tas, pdoy(tas, 20.0), window=3, freq=freq, bootstrap=True)
    exp = oracle(tas, t_x, B.spell_index("cold_spell_duration_index", 3, True, cal_max_doy=cmd), 20.0)
    np.testing.assert_array_equal(got.values, exp, err_msg="csdi")
    pp = pdoy(pr, 75.0)
    got = indices.days_over_precip_thresh(pr, pp, freq=freq, bootstrap=True)
    exp = oracle(pr, p_x, B.count_index(">", floor=1.0, cal_max_doy=cmd), 75.0)
    np.testing.assert_array_equal(got.values, exp, err_msg="days_over")
    got = indices.fraction_over_precip_thresh(pr, pp, freq=freq, bootstrap=True)
    exp = oracle(pr, p_x, B.fraction_index(1.0, cal_max_doy=cmd), 75.0, fraction=True)
    np.testing.assert_array_equal(got.values, exp, err_msg="fraction")


def test_unequal_block_loop_equals_fused(cuda):
    """_bootstrap_unequal_blocks on a noleap series (equal blocks) gives the fused kernels' bits."""
    import torch
    from xclim_b200 import _lib, bootstrapping as bs, device
    x, da = _series("noleap", list(range(2003, 2008)), 300, 3, "tas")
    from xclim_b200 import calendar as xcal
    per = xcal.select_percentile(xcal.percentile_doy(da.isel_time(da.time.sel_years(2004, 2006)), per=90.0), 90.0)
    b = bs._Setup(da, per, "MS")
    code = _lib.OPS[">"]
    for kind, rw, rbrl in (("spell", 6, True), ("spell", 3, False), ("count", 1, True)):
        fused, _ = device.bootstrap_doy_index(b.x2d, b.sl.start, b.N, b.L, b.step_period, b.P, b.window, b.percentile,
                                              b.alpha, b.beta, code, kind, rw, rbrl, 1.0 if kind == "count" else None)
        loop = bs._bootstrap_unequal_blocks(b.x2d, b.ta, b.sl, b.starts, b.lens, b.poff, b.step_period, b.window,
                                            b.percentile, b.alpha, b.beta,
                                            bs._replacement_index(kind, code, rw, rbrl, 1.0, None))
        m = torch.from_numpy(b.in_base).to(cuda)
        np.testing.assert_array_equal(fused[m].cpu().numpy(), loop[m].cpu().numpy(), err_msg=kind)


def test_unequal_block_loop_equals_fused_fraction(cuda):
    """The same cross-check for the fraction, whose loop takes the mean of the non-NaN float32 terms on the host."""
    import torch
    from xclim_b200 import _lib, bootstrapping as bs, calendar as xcal, device
    x, da = _series("noleap", list(range(2003, 2008)), 300, 4, "pr")
    x2 = x.copy()
    x2[::37, ::7] = np.inf                          # inf / inf: NaN fractions for some replacements
    da = make_field(x2, "2003-01-01", calendar="noleap", units="mm/d")
    per = xcal.select_percentile(xcal.percentile_doy(da.isel_time(da.time.sel_years(2004, 2006)), per=75.0), 75.0)
    b = bs._Setup(da, per, "MS")
    code = _lib.OPS[">"]
    table, doy_idx = b.table(per, da, 1.0)
    _, wet = device.period_sums_thr(b.x2d, b.poff, code, table, 1.0, doy_index=doy_idx)
    fused, _ = device.bootstrap_doy_index(b.x2d, b.sl.start, b.N, b.L, b.step_period, b.P, b.window, b.percentile,
                                          b.alpha, b.beta, code, "sum", 1, True, 1.0, wet)
    loop = bs._bootstrap_unequal_blocks(b.x2d, b.ta, b.sl, b.starts, b.lens, b.poff, b.step_period, b.window,
                                        b.percentile, b.alpha, b.beta,
                                        bs._replacement_index("sum", code, 1, True, 1.0, wet), fraction=True)
    m = torch.from_numpy(b.in_base).to(cuda)
    f, lp = fused[m].cpu().numpy(), loop[m].cpu().numpy()
    assert np.isnan(f).any() and np.isfinite(f).any()
    np.testing.assert_array_equal(f, lp)


def test_atmos_missing_and_streamed_input(cuda):
    """atmos.* with bootstrap=True: host-backed (streamed) input gives the device-resident result, and a period with
    a missing day is NaN (MissingAny)."""
    import torch
    from xclim_b200 import Field, atmos, calendar as xcal, indices
    x, _ = _series("noleap", list(range(2003, 2008)), 6 * 8, 5, "tas")
    x = x.reshape(x.shape[0], 6, 8)
    x[400, 2, 3] = np.nan                           # 2004-02-05: Feb 2004 of that cell
    host = make_field(x, "2003-01-01", calendar="noleap", units="K", dims=("time", "lat", "lon"))
    dev = Field(torch.from_numpy(x).to(cuda), host.dims, host.time, {}, dict(host.attrs))
    per = xcal.select_percentile(xcal.percentile_doy(host.isel_time(host.time.sel_years(2004, 2006)), per=90.0), 90.0)
    kw = dict(window=3, freq="MS", bootstrap=True)
    a = atmos.warm_spell_duration_index(host, per, **kw).values
    a = a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
    d = indices.warm_spell_duration_index(dev, per, **kw).values
    d = d.cpu().numpy() if hasattr(d, "cpu") else np.asarray(d)
    assert np.isnan(a[13, 2, 3])
    keep = np.ones(a.shape, bool)
    keep[13, 2, 3] = False
    np.testing.assert_array_equal(a[keep], d[keep])


@pytest.mark.parametrize("NB", [15, 30])
def test_full_size_wsdi(cuda, NB):
    """WSDI bootstrap on the (10950, 721, 1440) grid: mask offsets beyond 2^31, tiled when the masks do not fit.
    Sampled cells, the last 256 included, equal a small call on those cells alone; with the 15-year base two of
    them also equal the oracle."""
    import torch
    from xclim_b200 import _lib, device
    T, C, L = 10950, 721 * 1440, 365
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < 60e9:
        pytest.skip("needs 60 GB of free HBM")
    x = device.synth(T, C, kind=1, seed=5, cells_per_lat=1440, n_lat_global=721)
    sp = np.repeat(np.arange(NB), L).astype(np.int32)
    gt = _lib.OPS[">"]
    args = (NB, L, sp, NB, 5, 90.0, 1 / 3, 1 / 3, gt, "spell", 6, False)
    got, scratch = device.bootstrap_doy_index(x, 0, *args)
    del scratch
    cols = np.unique(np.r_[np.linspace(0, C - 257, 48).astype(np.int64), np.arange(C - 256, C)])
    cd = torch.from_numpy(cols).to(cuda)
    sub = x.index_select(1, cd).contiguous()
    small, _ = device.bootstrap_doy_index(sub, 0, *args)
    g = got.index_select(1, cd).cpu().numpy()
    np.testing.assert_array_equal(g, small.cpu().numpy())
    if NB == 15:
        two = [0, len(cols) - 1]
        exp, _ = fake_bootstrap.bootstrap_doy_index(torch.from_numpy(sub[:NB * L, two].cpu().numpy()), 0, *args)
        np.testing.assert_array_equal(g[:, two], exp.numpy())
    del x, got, sub
    torch.cuda.empty_cache()
