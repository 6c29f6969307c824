"""CPU tests of the percentile bootstrap of warm / cold spell duration, days over and fraction over a precipitation
percentile: the literal oracle, the host layer over the oracle-backed device stand-in (tests/fake_bootstrap.py), the
errors and the C argument checks."""
import ctypes

import numpy as np
import pytest

import fake_bootstrap
from oracle import bootstrap_oracle as B
from oracle import xclim_oracle as O
from xb_helpers import make_field


@pytest.fixture
def host(monkeypatch):
    fake_bootstrap.install(monkeypatch)


def _series(calendar, years, cells=2, seed=0, kind="tas"):
    rng = np.random.default_rng(seed)
    n = {"noleap": 365, "360_day": 360}.get(calendar)
    T = n * len(years) if n else int(sum(366 if (y % 4 == 0 and (y % 100 or y % 400 == 0)) else 365 for y in years))
    t = np.arange(T)
    if kind == "tas":
        x = 288 + 8 * np.sin(2 * np.pi * t / 365.25)[:, None] + 3 * rng.standard_normal((T, cells))
        x += 2.5 * np.repeat(rng.standard_normal((T // 4 + 1, cells)), 4, axis=0)[:T]    # multi-day spells
    else:
        x = rng.gamma(0.6, 5.0, (T, cells)) * (rng.random((T, cells)) < 0.5)
    x = x.astype(np.float32)
    return x, make_field(x, f"{years[0]}-01-01", calendar=calendar, units="K" if kind == "tas" else "mm/d")


def _pdoy(da, y0, y1, per, window=5):
    from xclim_b200 import calendar as xcal
    base = da.isel_time(da.time.sel_years(y0, y1))
    return xcal.select_percentile(xcal.percentile_doy(base, window=window, per=per), per)


def _feb29(da):
    return (np.asarray(da.time.month) == 2) & (np.asarray(da.time.day) == 29)


def label_years(da, freq):
    """Label year of every step's bootstrap year group, from the dates: the year in which a start-anchored group
    starts (YS: January, YS-JUL / QS-... / QS-DEC: the anchor month)."""
    anchor = {"YS": 1, "MS": 1, "QS-DEC": 12, "YS-JUL": 7}[freq]
    y, m = np.asarray(da.time.year), np.asarray(da.time.month)
    return np.where(m >= anchor, y, y - 1)


def _oracle(da, x, freq, base, index, per, fraction=False):
    t = da.time
    return B.bootstrap_doy_index(x, t.year, t.doy, t.bootstrap_group_ids(freq), label_years(da, freq),
                                 t.period_offsets(freq), base, index, window=5, per=per, feb29=_feb29(da),
                                 fraction=fraction)


@pytest.mark.parametrize("calendar", ["noleap", "standard"])
@pytest.mark.parametrize("freq", ["YS", "MS"])
def test_oracle_count_equals_bootstrap_doy_count(calendar, freq):
    """With the count index, the year-group oracle gives O.bootstrap_doy_count's bits (calendar-year groups)."""
    x, da = _series(calendar, list(range(2003, 2008)), seed=1)
    cmd = {"standard": 366, "noleap": 365, "360_day": 360}[calendar]
    got = _oracle(da, x, freq, (2004, 2006), B.count_index(">", cal_max_doy=cmd), 90.0)
    exp = O.bootstrap_doy_count(x, da.time.year, da.time.doy, da.time.period_offsets(freq), (2004, 2006), window=5,
                                per=90.0, op=">", cal_max_doy=cmd)
    np.testing.assert_array_equal(got, exp)


def test_fraction_mean_rule():
    v = np.array([[1.0, np.nan, np.nan], [2.0, 3.0, np.nan], [np.float32(0.1), 5.0, np.nan]], np.float32)
    out = B.fraction_mean(v)
    assert out[0] == np.float32((1.0 + 2.0 + float(np.float32(0.1))) / 3)
    assert out[1] == np.float32(4.0) and np.isnan(out[2])


@pytest.mark.parametrize("calendar", ["noleap", "standard"])
@pytest.mark.parametrize("freq,rbrl,window", [("YS", True, 6), ("MS", True, 3), ("MS", False, 3), ("YS", False, 1)])
def test_spell_indices_host(host, calendar, freq, rbrl, window):
    from xclim_b200 import indices
    x, da = _series(calendar, list(range(2003, 2008)), seed=2)
    cmd = {"standard": 366, "noleap": 365, "360_day": 360}[calendar]
    for name, per, op in (("warm_spell_duration_index", 80.0, ">"), ("cold_spell_duration_index", 20.0, "<")):
        pdoy = _pdoy(da, 2004, 2006, per)
        got = getattr(indices, name)(da, pdoy, window=window, freq=freq, resample_before_rl=rbrl, bootstrap=True)
        exp = _oracle(da, x, freq, (2004, 2006), B.spell_index(name, window, rbrl, cal_max_doy=cmd), per)
        np.testing.assert_array_equal(got.values, exp, err_msg=name)
        assert got.values.dtype == np.float64 and got.attrs["units"] == "d"


@pytest.mark.parametrize("calendar", ["noleap", "standard"])
@pytest.mark.parametrize("freq", ["YS", "MS"])
def test_precip_indices_host(host, calendar, freq):
    from xclim_b200 import indices
    x, da = _series(calendar, list(range(2003, 2007)), seed=3, kind="pr")
    cmd = {"standard": 366, "noleap": 365, "360_day": 360}[calendar]
    pdoy = _pdoy(da, 2004, 2005, 75.0)
    got = indices.days_over_precip_thresh(da, pdoy, thresh="1 mm/day", freq=freq, bootstrap=True)
    exp = _oracle(da, x, freq, (2004, 2005), B.count_index(">", floor=1.0, cal_max_doy=cmd), 75.0)
    np.testing.assert_array_equal(got.values, exp)
    got = indices.fraction_over_precip_thresh(da, pdoy, thresh="1 mm/day", freq=freq, bootstrap=True)
    exp = _oracle(da, x, freq, (2004, 2005), B.fraction_index(1.0, cal_max_doy=cmd), 75.0, fraction=True)
    np.testing.assert_array_equal(got.values, exp)
    assert got.values.dtype == np.float32


def test_spell_cut_at_out_of_base_year_edge(host):
    """resample_before_rl=False: a spell across the edge of an out-of-base year is split in two by bootstrap=True,
    as in the reference (each year is its own slice), and only there."""
    from xclim_b200 import indices
    x, da = _series("noleap", list(range(2003, 2008)), seed=4)
    pdoy = _pdoy(da, 2004, 2006, 90.0)
    x2 = x.copy()
    edge = 365 * 4                                   # 2007-01-01: out of base
    x2[edge - 3:edge + 3] = 400.0
    da2 = make_field(x2, "2003-01-01", calendar="noleap", units="K")
    a = indices.warm_spell_duration_index(da2, pdoy, window=6, freq="MS", resample_before_rl=False, bootstrap=True)
    b = indices.warm_spell_duration_index(da2, pdoy, window=6, freq="MS", resample_before_rl=False)
    exp = _oracle(da2, x2, "MS", (2004, 2006), B.spell_index("warm_spell_duration_index", 6, False), 90.0)
    np.testing.assert_array_equal(a.values, exp)
    dec06 = 12 * 3 + 11
    assert b.values[dec06, 0] >= 6 and a.values[dec06, 0] < b.values[dec06, 0]
    out = np.ones(a.values.shape[0], bool)
    out[12:48] = False
    out[dec06] = False
    np.testing.assert_array_equal(a.values[out & (np.arange(len(out)) >= 48)],
                                  b.values[out & (np.arange(len(out)) >= 48)].astype(np.float64))


@pytest.mark.parametrize("freq", ["YS-JUL", "QS-DEC"])
def test_in_base_groups_by_label_year(host, freq):
    """A year group is bootstrapped when its LABEL year is a base year (core/bootstrapping.py:184), over the whole
    group: with YS-JUL the group labelled 2003 (Jul 2003 - Jun 2004) keeps the plain value although it holds base
    days; with QS-DEC the group labelled 2006 (Dec 2006 - Nov 2007) is bootstrapped into 2007, and the one labelled
    2003 (Dec 2003 - Nov 2004) is not."""
    from xclim_b200 import indices
    x, da = _series("noleap", list(range(2003, 2008)), cells=4, seed=8, kind="pr")
    pdoy = _pdoy(da, 2004, 2006, 75.0)
    got = indices.days_over_precip_thresh(da, pdoy, freq=freq, bootstrap=True).values
    plain = indices.days_over_precip_thresh(da, pdoy, freq=freq).values.astype(np.float64)
    np.testing.assert_array_equal(got, _oracle(da, x, freq, (2004, 2006), B.count_index(">", floor=1.0, cal_max_doy=365),
                                               75.0))
    labels = da.time.period_labels(freq)
    lab = np.array([int(v[:4]) - (0 if int(v[5:7]) >= (7 if freq == "YS-JUL" else 12) else 1) for v in labels])
    boot = (lab >= 2004) & (lab <= 2006)
    np.testing.assert_array_equal(got[~boot], plain[~boot])
    assert (got[boot] != plain[boot]).any()
    first = labels.index("2003-07-01" if freq == "YS-JUL" else "2003-12-01")
    assert not boot[first]                          # holds base days (2004), label 2003: plain
    if freq == "QS-DEC":
        last = [labels.index(d) for d in ("2006-12-01", "2007-03-01", "2007-06-01", "2007-09-01")]
        assert boot[last].all()                     # Dec 2006 - Nov 2007, label 2006: bootstrapped
        assert (got[last] != plain[last]).any()


# the five rows of the reference's bootstrap test the package lacked (tests/test_bootstrapping.py:22-74)
ROWS = [(name, per, "MS", cal) for cal in ("noleap", "standard")
        for name, per in (("warm_spell_duration_index", 98), ("cold_spell_duration_index", 2),
                          ("days_over_precip_thresh", 99), ("fraction_over_precip_thresh", 98))]


@pytest.mark.parametrize("name,per,freq,calendar", ROWS)
def test_reference_property_rows(host, name, per, freq, calendar):
    """In-base values rise more often than they fall with bootstrap; out-of-base values equal the plain call."""
    from xclim_b200 import indices
    kind = "pr" if "precip" in name else "tas"
    x, da = _series(calendar, list(range(2000, 2006)), cells=3, seed=5, kind=kind)
    pdoy = _pdoy(da, 2001, 2003, float(per))
    kw = {"freq": freq}
    fn = getattr(indices, name)
    no = fn(da, pdoy, **kw).values.astype(np.float64)
    bo = fn(da, pdoy, bootstrap=True, **kw).values.astype(np.float64)
    yrs = np.repeat(np.arange(2000, 2006), 12)
    inb = (yrs >= 2001) & (yrs <= 2003)
    np.testing.assert_almost_equal(bo[~inb], no[~inb], 15)
    d = bo[inb] - no[inb]
    d = d[np.isfinite(d)]
    assert (d > 0).sum() > (d < 0).sum()            # tests/test_bootstrapping.py:69


def test_errors_in_reference_order(host):
    from xclim_b200 import Field, bootstrapping, indices
    x, da = _series("noleap", list(range(2003, 2007)), seed=6)
    pdoy = _pdoy(da, 2004, 2005, 90.0)
    bad = Field(np.asarray(pdoy.values), pdoy.dims, None, dict(pdoy.coords), {"units": "K"})
    for fn in (indices.warm_spell_duration_index, indices.cold_spell_duration_index):
        with pytest.raises(NotImplementedError, match="percentile_doy"):
            fn(da, bad, bootstrap=True, op="==")       # provenance first (core/bootstrapping.py:131-143)
    with pytest.raises(KeyError, match="percentile_doy"):
        indices.tx90p(da, bad, bootstrap=True)
    assert issubclass(bootstrapping.BootstrapPercentileError, (KeyError, NotImplementedError))
    for fn in (indices.days_over_precip_thresh, indices.fraction_over_precip_thresh):
        with pytest.raises(bootstrapping.BootstrapPercentileError):
            fn(da, bad, bootstrap=True)                # before the unit conversion of thresh
        per_cell = Field(np.ones(2), ("d0",), None, {}, {"units": "mm/d"})
        with pytest.raises(KeyError, match="percentile_doy"):
            fn(da, per_cell, bootstrap=True)
    p_all = _pdoy(da, 2003, 2006, 90.0)
    with pytest.raises(KeyError, match="all years are overlapping"):
        indices.warm_spell_duration_index(da, p_all, bootstrap=True)
    with pytest.raises(NotImplementedError, match="nest"):
        indices.warm_spell_duration_index(da, pdoy, freq="7D", bootstrap=True)
    with pytest.raises(ValueError, match="not permitted"):
        indices.warm_spell_duration_index(da, pdoy, bootstrap=True, op="<")


def test_abi_argument_checks():
    from xclim_b200 import _lib
    lib = _lib.load()
    f = lib.xc_bootstrap_doy_index_f32
    buf = (ctypes.c_uint32 * 64)()
    p = ctypes.addressof(buf)
    assert lib.xc_bootstrap_doy_index_scratch_bytes(15, 365, 10) == 15 * 14 * 12 * 4 * 10
    assert lib.xc_bootstrap_doy_index_scratch_bytes(1, 365, 10) == 0

    def call(**kw):
        a = dict(x=p, T=730, C=4, ldx=4, b0=0, N=2, L=365, sp=p, P=2, w=5, q=90.0, al=1 / 3, be=1 / 3, op=0, red=1,
                 rw=6, rb=1, fl=float("-inf"), wet=None, sc=p, sb=256, out=p)
        a.update(kw)
        r = f(a["x"], a["T"], a["C"], a["ldx"], a["b0"], a["N"], a["L"], a["sp"], a["P"], a["w"], a["q"], a["al"],
              a["be"], a["op"], a["red"], a["rw"], a["rb"], a["fl"], a["wet"], a["sc"], a["sb"], a["out"], None)
        return r, lib.xc_last_error().decode()
    assert call(x=None) == (-1, "null pointer argument")
    assert call(red=3)[1].startswith("unknown bootstrap index")
    assert call(op=4)[0] == -1
    assert call(rw=0)[1] == "run window must be >= 1"
    assert call(fl=float("nan"))[1] == "floor must not be NaN"
    assert call(fl=1.0, op=1)[1] == "a threshold floor needs op > or >="
    assert call(red=2)[1] == "wet_total is given exactly for XC_BOOT_SUM"
    assert call(wet=p)[1] == "wet_total is given exactly for XC_BOOT_SUM"
    assert call(sc=p + 4)[1] == "scratch must be 16-byte aligned"
    assert call(sb=16)[1].startswith("scratch of 16 bytes holds the masks of 0 cells")
    assert call(N=3)[1] == "base period outside the series"
    assert call(w=4)[1].startswith("window must be odd")
