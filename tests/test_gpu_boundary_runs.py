"""The three entry points of csrc/boundary.cu -- first / last run per period (`xc_period_boundary_run_f32`), runs
confined to a per-period range (`xc_period_boundary_run_range_f32`) and the quantile of the run lengths
(`xc_period_run_quantile_f32`) -- bit for bit against the reference-semantics oracle on hostile float data, every
operator, windows around the 8-row load chunk, irregular periods and grid edges; then the public indices built on
them, on three calendars and four frequencies."""
import numpy as np
import pytest

import fake_device as FD
from oracle import xclim_oracle as O
from xb_helpers import make_field
from xclim_b200 import _lib

pytestmark = pytest.mark.gpu

F32 = np.float32
FMAX = float(np.finfo(F32).max)
TINY = float(np.finfo(F32).smallest_subnormal)
OPS = (">", "<", ">=", "<=", "==", "!=")
WINDOWS = (1, 2, 7, 8, 9, 16, 17)
# (threshold, cmp_f64): float32 numbers, thresholds that are not (compared in float32 or in float64), a subnormal,
# the float32 extremes and a float64 threshold beyond them
THRESHOLDS = [(0.0, 0), (0.1, 0), (0.1, 1), (-1e-40, 1), (-1e-40, 0), (3.4e38, 0), (3.4e38, 1), (1e39, 1)]


def _palette(thr, cmp_f64):
    """The threshold, its float32 neighbours (those of both directed roundings for a float64 threshold) and the
    hostile values: NaN, +-inf, +-0, subnormals, +-3.4e38, the float32 extremes."""
    with np.errstate(over="ignore"):
        t = F32(thr)
        vals = [t, np.nextafter(t, F32(np.inf)), np.nextafter(t, F32(-np.inf))]
        if cmp_f64:
            vals += [np.nextafter(v, F32(s)) for v in vals for s in (np.inf, -np.inf)]
    vals += [np.nan, np.inf, -np.inf, 0.0, -0.0, TINY, -TINY, 1e-40, 3.4e38, -3.4e38, FMAX, -FMAX, 1.0, -1.0, 2.5]
    return np.array(vals, F32)


def _true_false(pal, op, thr, cmp_f64):
    """A value the condition holds on and a non-NaN one it fails on (the other one where no such value exists, such
    as == against a threshold float32 cannot hold)."""
    c = FD._cond(pal, _lib.OPS[op], np.float64(thr) if cmp_f64 else thr, cmp_f64)
    f = ~c & ~np.isnan(pal)
    tv = pal[c][0] if c.any() else pal[f][0]
    fv = pal[f][0] if f.any() else tv
    return tv, fv


def _poff_months(first, last, n_years=1):
    """Irregular month lengths with a partial first and last period."""
    lens = [first] + [31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31] * n_years + [last]
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


def _data(rng, poff, C, pal, tv, fv):
    """Persistent draws from the palette (runs across period edges, runs cut by the series ends), then planted
    columns: all-True, all-False, all-NaN, runs of window-like lengths starting at each position of an 8-row chunk
    from the period start, runs ending on the period's last step, runs crossing the period end, NaN-broken runs and
    periods that are True throughout."""
    T = int(poff[-1])
    flip = rng.choice([0.02, 0.1, 0.4], size=C)
    flips = rng.random((T, C)) < flip
    flips[0] = True
    vals = rng.choice(pal, size=(T, C))
    idx = np.maximum.accumulate(np.where(flips, np.arange(T)[:, None], 0), axis=0)
    x = vals[idx, np.arange(C)]
    if C < 48:
        if C >= 3:
            x[:, 0], x[:, 1], x[:, 2] = tv, fv, np.nan
        return x
    base = C - 48                            # the planted columns sit at the end: in the last CTA on wide grids
    x[:, base:] = fv
    x[:, base + 0] = tv
    x[:, base + 2] = np.nan
    lens = (1, 2, 7, 8, 9, 16, 17)
    for p in range(len(poff) - 1):
        t0, t1 = int(poff[p]), int(poff[p + 1])
        for j in range(18):                  # run of lens[j % 7] steps from t0 + (j % 9)
            s = t0 + j % 9
            x[s:min(T, s + lens[j % 7]), base + 3 + j] = tv
        for j in range(7):                   # run ending on t1 - 1
            x[max(0, t1 - lens[j]):t1, base + 21 + j] = tv
        for j in range(7):                   # run from t1 - 1 - j crossing into the next period by j + 1 steps
            x[max(0, t1 - 1 - j):min(T, t1 + 1 + j), base + 28 + j] = tv
        if p % 2 == 0:
            x[t0:t1, base + 35] = tv         # True throughout the period, False in the next
            x[t0:t1, base + 36] = tv
            x[t0:t1:5, base + 36] = np.nan   # broken by NaN every 5 steps
    x[:, base + 37] = np.where(np.arange(T) % 9 == 4, np.nan, tv)
    return x


def _dev(x, cuda):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).to(cuda)


def _eq(got, exp, msg=""):
    """Bit for bit (any NaN matches any NaN; the outputs are small integers, lengths or NaN)."""
    got = got.cpu().numpy() if hasattr(got, "cpu") else np.asarray(got)
    exp = np.asarray(exp).astype(F32)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(exp), err_msg=f"{msg}: NaN positions")
    bad = (got.view(np.uint32) != exp.view(np.uint32)) & ~np.isnan(exp)
    assert not bad.any(), f"{msg}: {int(bad.sum())} differ, first at {np.argwhere(bad)[0]}: " \
                          f"{got[tuple(np.argwhere(bad)[0])]} vs {exp[tuple(np.argwhere(bad)[0])]}"


# ------------------------------------------------------------------------------ xc_period_boundary_run_f32
@pytest.mark.parametrize("thr,cmp_f64", THRESHOLDS)
@pytest.mark.parametrize("op", OPS)
def test_boundary_run_operators_and_windows(cuda, op, thr, cmp_f64):
    from xclim_b200 import device
    rng = np.random.default_rng(OPS.index(op) * 100 + THRESHOLDS.index((thr, cmp_f64)))
    poff = _poff_months(17, 9)
    pal = _palette(thr, cmp_f64)
    tv, fv = _true_false(pal, op, thr, cmp_f64)
    x = _data(rng, poff, 129, pal, tv, fv)
    cond = FD._cond(x, _lib.OPS[op], np.float64(thr) if cmp_f64 else thr, cmp_f64)
    xd = _dev(x, cuda)
    for w in WINDOWS:
        for last, ofn in ((False, O.first_run), (True, O.last_run)):
            got = device.period_boundary_run(xd, poff, _lib.OPS[op], thr, w, last=last, cmp_f64=cmp_f64)
            _eq(got, ofn(cond, w, poff=poff), f"{op} {thr} f64={cmp_f64} w={w} last={last}")


def _periods(kind, rng):
    if kind == "one_step":
        return np.arange(61, dtype=np.int32)
    if kind == "months":
        return _poff_months(5, 20, n_years=2)
    if kind == "whole":
        return np.array([0, 300], np.int32)
    lens = rng.integers(1, 14, size=300)                         # a few hundred periods of 1 to 13 steps
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


@pytest.mark.parametrize("kind", ["one_step", "months", "whole", "many"])
def test_boundary_run_period_shapes(cuda, kind):
    """Windows around the period length and beyond the series, on one-step periods, months, P = 1 and ~300
    periods."""
    from xclim_b200 import device
    rng = np.random.default_rng(len(kind))
    poff = _periods(kind, rng)
    T = int(poff[-1])
    plen = int(np.max(np.diff(poff)))
    for op in (">", "!="):
        pal = _palette(0.5, 0)
        tv, fv = _true_false(pal, op, 0.5, 0)
        x = _data(rng, poff, 130, pal, tv, fv)
        cond = FD._cond(x, _lib.OPS[op], 0.5)
        xd = _dev(x, cuda)
        for w in sorted({1, 2, 8, 9, 17, plen, plen + 1, T, T + 1}):
            for last, ofn in ((False, O.first_run), (True, O.last_run)):
                got = device.period_boundary_run(xd, poff, _lib.OPS[op], 0.5, w, last=last)
                _eq(got, ofn(cond, w, poff=poff), f"{kind} {op} w={w} last={last}")


def _views(x, cuda):
    """The contiguous buffer, a column slice at a 4-byte offset with ldx = C + 1, and one with ldx >> C."""
    T, C = x.shape
    a = np.full((T, C + 1), 7.0, F32)
    a[:, 1:] = x
    b = np.full((T, 4 * C + 37), -7.0, F32)
    b[:, 5:5 + C] = x
    return {"contiguous": _dev(x, cuda), "ldx=C+1": _dev(a, cuda)[:, 1:], "ldx>>C": _dev(b, cuda)[:, 5:5 + C]}


@pytest.mark.parametrize("C", [1, 3, 127, 128, 129, 300, 4100])
def test_boundary_entry_points_on_grid_edges_and_views(cuda, C):
    """Every view gives the contiguous call's bits, and those are the oracle's, for all three entry points."""
    from xclim_b200 import device
    rng = np.random.default_rng(C)
    poff = np.array([0, 3, 31, 59, 90, 95, 96, 140], np.int32)
    pal = _palette(0.0, 0)
    tv, fv = _true_false(pal, ">", 0.0, 0)
    x = _data(rng, poff, C, pal, tv, fv)
    views = _views(x, cuda)
    assert views["ldx=C+1"].stride(0) == C + 1 and views["ldx>>C"].stride(0) == 4 * C + 37
    P = len(poff) - 1
    mid = rng.integers(0, np.diff(poff))
    lo = np.where(np.arange(P) % 4 == 3, -1, poff[:-1] + mid).astype(np.int32)
    hi = poff[1:].astype(np.int32)
    for op in (">", "!="):
        code = _lib.OPS[op]
        cond = FD._cond(x, code, 0.0)
        exp = {}
        for w, last in ((1, False), (8, False), (9, True)):
            fn = O.last_run if last else O.first_run
            exp[("run", w, last)] = (lambda xd, w=w, last=last: device.period_boundary_run(xd, poff, code, 0.0, w, last),
                                     fn(cond, w, poff=poff))
            exp[("range", w, last)] = (
                lambda xd, w=w, last=last: device.period_boundary_run_range(xd, poff, lo, hi, code, 0.0, w, last=last),
                _range_oracle(cond, poff, lo, hi, w, last))
        for q, w, before in ((0.5, 1, True), (0.9, 2, False)):
            exp[("q", q, w, before)] = (
                lambda xd, q=q, w=w, before=before: device.period_run_quantile(xd, poff, code, 0.0, q, w, before),
                O.resample_and_rl(cond, before, O.rle_statistics, poff=poff, reducer=q, window=w))
        for key, (call, ref) in exp.items():
            base = call(views["contiguous"])
            _eq(base, ref, f"C={C} {op} {key}")
            for name in ("ldx=C+1", "ldx>>C"):
                got = call(views[name])
                assert np.array_equal(got.cpu().numpy().view(np.uint32), base.cpu().numpy().view(np.uint32)), \
                    f"C={C} {op} {key} {name}"


# ------------------------------------------------------------------------------ xc_period_boundary_run_range_f32
def _range_oracle(cond, poff, lo, hi, window, last=False, negate=False, cell_lo=None):
    """The reference's composition per group: the condition masked to [lo, hi) (and to index >= cell_lo.fillna(0))
    with NaN, then first_run / last_run on the group (indices/run_length.py:977, 1148-1331)."""
    P, C = len(poff) - 1, cond.shape[1]
    out = np.full((P, C), np.nan)
    for p in range(P):
        t0, t1 = int(poff[p]), int(poff[p + 1])
        if lo[p] < 0:
            continue
        g = ~cond[t0:t1] if negate else cond[t0:t1]
        idx = np.arange(t1 - t0)[:, None]
        keep = (idx >= int(lo[p]) - t0) & (idx < int(hi[p]) - t0) & np.ones((1, C), bool)
        if cell_lo is not None:
            keep &= idx >= np.where(np.isnan(cell_lo[p]), 0, cell_lo[p])[None, :]
        out[p] = O.boundary_run(np.where(keep, g, np.nan), window, "last" if last else "first")
    return out


def _random_ranges(rng, poff, w):
    """Per period: the date absent (-1), the full period, after / up to / before a date, an empty range, a range
    clipped by the period end (hi > t1) and one starting before the period (lo < t0)."""
    P = len(poff) - 1
    lo, hi = poff[:-1].copy(), poff[1:].copy()
    for p in range(P):
        t0, t1 = int(poff[p]), int(poff[p + 1])
        mid = t0 + int(rng.integers(0, t1 - t0))
        kind = p % 8
        if kind == 0:
            lo[p] = -1
        elif kind == 2:
            lo[p] = mid                                   # time >= date
        elif kind == 3:
            hi[p] = mid + 1                               # time <= date
        elif kind == 4:
            hi[p] = min(mid + w - 1, t1)                  # time < date + window - 1
        elif kind == 5:
            lo[p], hi[p] = mid, mid                       # empty
        elif kind == 6:
            lo[p], hi[p] = mid, t1 + 3                    # clipped
        elif kind == 7:
            lo[p] = max(0, t0 - 2)                        # before the period: the period start
    return lo.astype(np.int32), hi.astype(np.int32)


def _cell_lo(rng, poff, lo, hi, C):
    """(P, C) float32 lower bounds relative to the period start: NaN, 0, inside the range, at hi, beyond hi."""
    P = len(poff) - 1
    out = np.zeros((P, C), F32)
    for p in range(P):
        t0 = int(poff[p])
        a, b = max(int(lo[p]), t0) - t0, int(hi[p]) - t0
        choice = rng.integers(0, 5, size=C)
        inside = rng.integers(a, max(a + 1, b), size=C)
        out[p] = np.select([choice == 0, choice == 1, choice == 2, choice == 3], [np.nan, 0, inside, b], b + 4)
    return out


@pytest.mark.parametrize("op", OPS)
def test_boundary_run_range_against_oracle(cuda, op):
    from xclim_b200 import device
    rng = np.random.default_rng(OPS.index(op) + 100)
    poff = _poff_months(13, 22, n_years=2)
    pal = _palette(0.0, 0)
    tv, fv = _true_false(pal, op, 0.0, 0)
    C = 131
    x = _data(rng, poff, C, pal, tv, fv)
    code = _lib.OPS[op]
    cond = FD._cond(x, code, 0.0)
    xd = _dev(x, cuda)
    for w in (1, 2, 8, 9, 17):
        lo, hi = _random_ranges(rng, poff, w)
        clo = _cell_lo(rng, poff, lo, hi, C)
        for last in (False, True):
            for negate in (False, True):
                for cl in (None, clo):
                    got = device.period_boundary_run_range(xd, poff, lo, hi, code, 0.0, w, last=last, negate=negate,
                                                           cell_lo=None if cl is None else _dev(cl, cuda))
                    what = f"{op} w={w} last={last} negate={negate} cell_lo={cl is not None}"
                    _eq(got, _range_oracle(cond, poff, lo, hi, w, last, negate, cl), what)
                    if w in (1, 9) and not last:     # the literal restatement of the ABI contract, on a sample
                        _eq(got, FD.period_boundary_run_range(x, poff, lo, hi, code, 0.0, w, last, negate, cl), what)


@pytest.mark.parametrize("mid_date", ["01-01", "03-01", "07-01", "12-31"])
def test_boundary_run_range_named_modes(cuda, mid_date):
    """Ranges from seasons._ranges on a real axis (the date absent from some groups, on the first or the last
    step of others) against the per-group oracle functions."""
    from xclim_b200 import TimeAxis, device, seasons
    rng = np.random.default_rng(len(mid_date) + int(mid_date[:2]))
    ta = TimeAxis.daily("2001-05-20", 365 * 3, "noleap")
    freq = "YS-JUL" if mid_date == "03-01" else "YS"
    poff = ta.period_offsets(freq)
    mids = [int(m) - int(s) if m >= 0 else None for m, s in zip(ta.date_index_in_periods(freq, mid_date), poff[:-1])]
    assert None in mids and any(m is not None for m in mids)
    pal = _palette(0.0, 0)
    tv, fv = _true_false(pal, "<", 0.0, 0)
    x = _data(rng, poff, 130, pal, tv, fv)
    code = _lib.OPS["<"]
    cond = FD._cond(x, code, 0.0)
    xd = _dev(x, cuda)

    def per_group(fn, c, w, **kw):
        return np.stack([fn(c[s:e], w, mids[p], **kw) for p, (s, e) in enumerate(O._groups(poff))])
    for w in (1, 3, 8, 9):
        cases = [("after", False, False, O.first_run_after_date, cond), ("before_incl", True, False,
                                                                          O.last_run_before_date, cond),
                 ("start", False, False, O.first_run_before_date, cond), ("after", False, True,
                                                                          O.first_run_after_date, ~cond)]
        for mode, last, negate, fn, c in cases:
            lo, hi = seasons._ranges(ta, freq, mid_date, mode, w)
            got = device.period_boundary_run_range(xd, poff, lo, hi, code, 0.0, w, last=last, negate=negate)
            _eq(got, per_group(fn, c, w), f"{mid_date} {mode} w={w} negate={negate}")
            _eq(got, FD.period_boundary_run_range(x, poff, lo, hi, code, 0.0, w, last, negate), f"{mode} restated")
        lo_a, hi_a = seasons._ranges(ta, freq, mid_date, "after", w)
        lo_b, hi_b = seasons._ranges(ta, freq, mid_date, "before_excl", w)
        end = device.period_boundary_run_range(xd, poff, lo_a, hi_a, code, 0.0, w, negate=True)
        beg = device.period_boundary_run_range(xd, poff, lo_b, hi_b, code, 0.0, w)
        _eq(beg, per_group(lambda g, w_, m: O.first_run_before_date(g, w_, m - w_ + 1) if m is not None else
                           np.full(g.shape[1:], np.nan), cond, w), f"before_excl w={w}")
        n = np.diff(poff).astype(F32)[:, None]
        e, b = end.cpu().numpy(), beg.cpu().numpy()
        e = np.where(np.isnan(b), np.nan, np.where(np.isnan(e) & ~np.isnan(b), n - 1, e))
        _eq(e, per_group(O.run_end_after_date, cond, w), f"run_end_after_date w={w}")
        lo_s, hi_s = seasons._ranges(ta, freq, mid_date, "start", w)
        beg = device.period_boundary_run_range(xd, poff, lo_s, hi_s, code, 0.0, w)
        end = device.period_boundary_run_range(xd, poff, lo_a, hi_a, code, 0.0, w, negate=True, cell_lo=beg)
        exp = [O.season_group(cond[s:e_], w, mids[p]) for p, (s, e_) in enumerate(O._groups(poff))]
        _eq(beg, np.stack([r[0] for r in exp]), f"season start w={w}")
        e = end.cpu().numpy()
        b = beg.cpu().numpy()
        e = np.where(np.isnan(b), np.nan, np.where(np.isnan(e) & ~np.isnan(b), n - 1, e))
        _eq(e, np.stack([r[1] for r in exp]), f"season end w={w}")


# ------------------------------------------------------------------------------ xc_period_run_quantile_f32
QS = (0.0, 0.05, 0.1, 0.5, 0.9, 0.999, 1.0)


def _rl_quantiles(cond, poff, before, qs, window):
    """{q: O.resample_and_rl(cond, before, O.rle_statistics, poff=poff, reducer=q, window=window)}, with the run
    lengths (O.rle) computed once for all q."""
    groups = O._groups(poff)
    if before:
        ds = [O.rle(cond[s:e]) for s, e in groups]
    else:
        d = O.rle(cond)
        ds = [d[s:e] for s, e in groups]
    return {q: np.stack([O._get_rl_stat(d, window, q) for d in ds]) for q in qs}


@pytest.mark.parametrize("before", [True, False])
@pytest.mark.parametrize("op,thr,cmp_f64", [(">", 0.0, 0), ("<", 0.1, 1), (">=", -1e-40, 0), ("<=", 3.4e38, 1),
                                            ("==", 0.0, 0), ("!=", 0.1, 1)])
def test_run_quantile_against_oracle(cuda, op, thr, cmp_f64, before):
    """The kernel equals the float64 oracle rounded to float32, with no tolerance: numpy's linear quantile is the
    lerp the kernel does.  Runs carried in from the previous period (skipped with resample_before_rl=False) and
    runs continuing to the series end are planted by _data."""
    from xclim_b200 import device
    rng = np.random.default_rng(OPS.index(op) * 2 + before)
    poff = _poff_months(10, 25)
    pal = _palette(thr, cmp_f64)
    tv, fv = _true_false(pal, op, thr, cmp_f64)
    x = _data(rng, poff, 129, pal, tv, fv)
    x[-40:, ::3] = tv                                        # runs cut by the end of the series
    cond = FD._cond(x, _lib.OPS[op], np.float64(thr) if cmp_f64 else thr, cmp_f64)
    xd = _dev(x, cuda)
    for w in (1, 2, 5):
        exp = _rl_quantiles(cond, poff, before, QS, w)
        if w == 2 and not before:
            np.testing.assert_array_equal(exp[0.5], O.resample_and_rl(cond, before, O.rle_statistics, poff=poff,
                                                                      reducer="q5", window=w))
        for q in QS:
            got = device.period_run_quantile(xd, poff, _lib.OPS[op], thr, q, w, before, cmp_f64=cmp_f64)
            _eq(got, exp[q], f"{op} {thr} q={q} w={w} before={before}")


def _max_period():
    """The longest period the host's shared-memory check (xc_period_run_quantile_f32) accepts."""
    ok = lambda L: (L // 2 + 2) * 128 * 2 <= 200 * 1024   # noqa: E731  (cap = len / 2 + 2 uint16 per lane)
    L = 1
    while ok(L + 1):
        L += 1
    return L


@pytest.mark.parametrize("T", [1000, "max"])
def test_run_quantile_shared_memory_opt_in(cuda, T):
    """freq=None: one period of T steps, above the 48 KiB default of dynamic shared memory, up to the size limit."""
    from xclim_b200 import device
    T = _max_period() if T == "max" else T
    rng = np.random.default_rng(T)
    poff = np.array([0, T], np.int32)
    x = _data(rng, poff, 130, _palette(0.0, 0), F32(1.0), F32(-1.0))
    x[:, 5] = np.where(np.arange(T) % 2 == 0, 1.0, -1.0)      # the most runs a period can hold
    cond = FD._cond(x, _lib.OPS[">"], 0.0)
    xd = _dev(x, cuda)
    for q in (0.0, 0.5, 0.999, 1.0):
        for w in (1, 2):
            got = device.period_run_quantile(xd, poff, _lib.OPS[">"], 0.0, q, w, True)
            _eq(got, O.rle_statistics(cond, q, w)[None], f"T={T} q={q} w={w}")


def test_run_quantile_size_limit_raises(cuda):
    import torch

    from xclim_b200 import device
    L = _max_period() + 1
    x = torch.zeros((L, 4), device=cuda)
    with pytest.raises(NotImplementedError, match="too many runs"):
        device.period_run_quantile(x, np.array([0, L], np.int32), _lib.OPS[">"], 0.0, 0.5, 1)
    with pytest.raises(NotImplementedError, match="too many runs"):     # the longest period decides
        device.period_run_quantile(torch.zeros((L + 1, 4), device=cuda), [0, 1, L + 1], _lib.OPS[">"], 0.0, 0.5, 1)
    device.period_run_quantile(x, [0, 1, L], _lib.OPS[">"], 0.0, 0.5, 1)   # L - 1 steps: accepted
    torch.cuda.synchronize()


def test_run_quantile_run_longer_than_65535(cuda):
    """A run of more than 65535 steps attributed with its full length to the period where it starts
    (resample_before_rl=False), beside ordinary cells; also through rle_statistics(freq="YS")."""
    from xclim_b200 import device
    from xclim_b200 import run_length as rl
    T = 70000
    rng = np.random.default_rng(65536)
    m = rng.random((T, 6)) < 0.6
    m[:, 0] = True                                      # one run of T steps
    m[:, 1] = True
    m[:400, 1] = rng.random(400) < 0.5                  # short runs, then a run of 69600+ steps from period 1
    m[200:, 2] = True                                   # a run from inside period 0 to the end
    m[:, 3] = False
    da = make_field(m, "1850-01-01", calendar="noleap", units="")
    poff = da.time.period_offsets("YS")
    xd = _dev(m.astype(F32), cuda)
    for q in (0.0, 0.5, 1.0):
        for w in (1, 3):
            got = device.period_run_quantile(xd, poff, _lib.OPS[">"], 0.0, q, w, False)
            exp = O.rle_statistics(m, q, w, poff=poff)
            _eq(got, exp, f"q={q} w={w}")
    got = rl.rle_statistics(da, "q50", 1, freq="YS").values
    _eq(got, O.rle_statistics(m, "q50", 1, poff=poff), "rle_statistics q50 YS")
    assert got[0, 0] == T
    got = rl.rle_statistics(da, "q90", 2, freq="YS", index="last").values
    _eq(got, O.rle_statistics(m, "q90", 2, poff=poff, index="last"), "rle_statistics q90 YS last")
    assert got[-1, 0] == T


# ------------------------------------------------------------------------------ the public indices
CALENDARS = {"noleap": ("2001-03-15", 1100), "standard": ("1999-08-20", 1150), "360_day": ("2001-09-01", 1000)}


def _tas(rng, T, shape):
    t = np.arange(T)
    x = 279 + 12 * np.sin(2 * np.pi * (t % 365 - 110) / 365)[(slice(None),) + (None,) * len(shape)]
    x = (x + 5 * rng.standard_normal((T,) + shape)).astype(F32)
    x[rng.random(x.shape) < 0.004] = np.nan
    return x


def _doy(v, poff, ta):
    t = np.where(np.isnan(v), 0, v).astype(int) + np.asarray(poff[:-1]).reshape((-1,) + (1,) * (v.ndim - 1))
    return np.where(np.isnan(v), np.nan, np.asarray(ta.doy)[t])


@pytest.mark.parametrize("calendar,freq", [("noleap", "YS"), ("noleap", "MS"), ("standard", "YS-JUL"),
                                           ("standard", "QS-DEC"), ("360_day", "YS"), ("360_day", "QS-DEC")])
def test_public_run_indices(cuda, calendar, freq):
    """first_run / last_run (both coords, 0/1/NaN float masks), the q-reducers of rle_statistics (index first /
    last, freq and None) and resample_and_rl, first / last_occurrence (str, float and float64 thresholds)."""
    from xclim_b200 import generic
    from xclim_b200 import run_length as rl
    start, T = CALENDARS[calendar]
    rng = np.random.default_rng(len(calendar) * 10 + len(freq))
    shape = (3, 43)
    mf = (rng.random((T,) + shape) < 0.6).astype(F32)
    mf[rng.random(mf.shape) < 0.02] = np.nan
    mf[:, 0, 0], mf[:, 0, 1] = 1.0, 0.0
    da = make_field(mf, start, calendar=calendar, units="")
    ta = da.time
    poff = ta.period_offsets(freq)
    for w in (1, 2, 9):
        for fn, ofn in ((rl.first_run, O.first_run), (rl.last_run, O.last_run)):
            idx = ofn(mf, w, poff=poff)
            np.testing.assert_array_equal(fn(da, w, freq=freq).values, idx, err_msg=f"{fn.__name__} w={w}")
            np.testing.assert_array_equal(fn(da, w, freq=freq, coord="dayofyear").values, _doy(idx, poff, ta),
                                          err_msg=f"{fn.__name__} doy w={w}")
    m = rng.random((T,) + shape) < 0.7
    dm = make_field(m, start, calendar=calendar, units="")
    for red, w in (("q05", 1), ("q5", 2), ("q90", 5), ("q999", 1)):
        for index in ("first", "last"):
            got = rl.rle_statistics(dm, red, w, freq=freq, index=index).values
            _eq(got, O.rle_statistics(m, red, w, poff=poff, index=index), f"{red} w={w} {index}")
        _eq(rl.rle_statistics(dm, red, w).values, O.rle_statistics(m, red, w), f"{red} w={w} freq=None")
        for before in (True, False):
            got = rl.resample_and_rl(dm, before, rl.rle_statistics, reducer=red, window=w, freq=freq).values
            exp = O.resample_and_rl(m, before, O.rle_statistics, poff=poff, reducer=red, window=w)
            _eq(got, exp, f"resample_and_rl {red} w={w} before={before}")
    x = _tas(rng, T, shape)
    on = rng.random(x.shape) < 0.05                 # on the threshold in float32, where float64 compares differ
    x[on] = rng.choice(np.array([278.15, 300.0, np.nextafter(F32(278.15), F32(0))], F32), size=int(on.sum()))
    xa = make_field(x, start, calendar=calendar, units="K")
    for thr, oth in (("5 degC", 278.15), (278.15, 278.15), (np.float64(278.15), np.float64(278.15)), (300, 300.0)):
        for op in (">=", "<", "!="):
            cond = O.compare(x, op, oth)
            for fn, ofn in ((generic.first_occurrence, O.first_run), (generic.last_occurrence, O.last_run)):
                got = fn(xa, thr, freq, op).values
                np.testing.assert_array_equal(got, _doy(ofn(cond, 1, poff=poff), poff, ta),
                                              err_msg=f"{fn.__name__} {thr!r} {op}")


@pytest.mark.parametrize("freq", ["YS", "YS-JUL", "MS", "QS-DEC"])
@pytest.mark.parametrize("calendar", list(CALENDARS))
def test_public_season_indices(cuda, calendar, freq):
    """generic.season (three stats, mid_date None or a date absent from some groups), first_day_threshold_reached,
    last_spring_frost, run_end_after_date and the growing / frost / frost-free season indices."""
    from xclim_b200 import generic, indices, seasons
    from xclim_b200.generic import _unwrap
    start, T = CALENDARS[calendar]
    rng = np.random.default_rng(len(calendar) + 7 * len(freq))
    shape = (3, 43)
    x = _tas(rng, T, shape)
    x[:, 0, 0], x[:, 0, 1] = 300.0, 200.0
    da = make_field(x, start, calendar=calendar, units="K")
    ta = da.time
    poff = ta.period_offsets(freq)

    def mids_of(date):
        if date is None:
            return [None] * (len(poff) - 1)
        return [int(m) - int(s) if m >= 0 else None for m, s in zip(ta.date_index_in_periods(freq, date), poff[:-1])]

    def per_group(fn, cond, w, date):
        mids = mids_of(date)
        return _doy(np.stack([fn(cond[s:e], w, mids[p]) for p, (s, e) in enumerate(O._groups(poff))]), poff, ta)

    def season(cond, w, date, stat):
        return O.season(cond, w, mids_of(date), poff, stat, ta.doy, has_date=date is not None)

    ge = O.compare(x, ">=", 278.15)
    for mid in (None, "07-01", "01-01"):
        for w in (1, 5):
            for stat in ("start", "end", "length"):
                got = generic.season(da, "5 degC", w, ">=", stat, freq, mid_date=mid).values
                np.testing.assert_array_equal(got, season(ge, w, mid, stat), err_msg=f"season {stat} {mid} w={w}")
    lt = O.compare(x, "<", 273.15)
    gt = O.compare(x, ">", 273.15)
    x2d = _unwrap(da)[0]
    for w in (1, 3, 9):
        got = generic.first_day_threshold_reached(da, threshold="0 degC", op="<", after_date="07-01", window=w,
                                                  freq=freq).values
        np.testing.assert_array_equal(got, per_group(O.first_run_after_date, lt, w, "07-01"), err_msg=f"fdtr w={w}")
        got = indices.first_day_temperature_above(da, after_date="03-01", window=w, freq=freq).values
        np.testing.assert_array_equal(got, per_group(O.first_run_after_date, gt, w, "03-01"), err_msg=f"fdta w={w}")
        got = indices.last_spring_frost(da, window=w, freq=freq).values
        np.testing.assert_array_equal(got, per_group(O.last_run_before_date, lt, w, "07-01"), err_msg=f"lsf w={w}")
        got = seasons.run_end_after_date(x2d, ta, freq, _lib.OPS["<"], 273.15, w, "07-01").cpu().numpy()
        np.testing.assert_array_equal(got.reshape((-1,) + x.shape[1:]),
                                      per_group(O.run_end_after_date, lt, w, "07-01"), err_msg=f"run_end w={w}")
    for name, op, thr, w, mid, stat in (("growing_season_start", ">=", 278.15, 5, "07-01", "start"),
                                        ("growing_season_end", ">", 278.15, 5, "07-01", "end"),
                                        ("growing_season_length", ">=", 278.15, 6, "07-01", "length"),
                                        ("frost_season_length", "<", 273.15, 5, "01-01", "length"),
                                        ("frost_free_season_start", ">=", 273.15, 5, "07-01", "start"),
                                        ("frost_free_season_end", ">=", 273.15, 5, "07-01", "end"),
                                        ("frost_free_season_length", ">=", 273.15, 5, "07-01", "length")):
        got = getattr(indices, name)(da, freq=freq).values
        np.testing.assert_array_equal(got, season(O.compare(x, op, thr), w, mid, stat), err_msg=name)
