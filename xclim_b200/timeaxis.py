"""Daily time axis, calendars and ``resample(time=freq)`` period boundaries (host logic).

The reference delegates all of this to xarray/pandas/cftime (``da.resample(time=freq)``,
``time.dt.dayofyear`` ...; e.g. indices/generic.py:114, core/calendar.py:450-457).  The kernels only
need three small integer arrays per time axis -- period offsets, day-of-year index and a group
(year) index -- so this module computes them directly for the CF calendars, without xarray.  When an
``xarray.DataArray`` is passed in, :func:`TimeAxis.from_xarray` reads the same fields from
``da.time.dt`` instead, so any calendar xarray supports works.
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field

import numpy as np

_MONTHS = ["JAN", "FEB", "MAR", "APR", "MAY", "JUN", "JUL", "AUG", "SEP", "OCT", "NOV", "DEC"]
_DPM_NOLEAP = np.array([31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31])
_DPM_LEAP = np.array([31, 29, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31])

#: ``max_doy`` table of the reference (core/calendar.py:56-66).
MAX_DOY = {"standard": 366, "gregorian": 366, "proleptic_gregorian": 366, "julian": 366,
           "noleap": 365, "365_day": 365, "all_leap": 366, "366_day": 366, "360_day": 360}


def _is_leap(year: np.ndarray, calendar: str) -> np.ndarray:
    year = np.asarray(year)
    if calendar in ("noleap", "365_day", "360_day"):
        return np.zeros(year.shape, bool)
    if calendar in ("all_leap", "366_day"):
        return np.ones(year.shape, bool)
    if calendar == "julian":
        return year % 4 == 0
    return (year % 4 == 0) & ((year % 100 != 0) | (year % 400 == 0))


def _year_fields(year: int, calendar: str):
    """(month, day, doy) arrays for every day of ``year``."""
    if calendar == "360_day":
        month = np.repeat(np.arange(1, 13), 30)
        day = np.tile(np.arange(1, 31), 12)
    else:
        dpm = _DPM_LEAP if bool(_is_leap(np.array(year), calendar)) else _DPM_NOLEAP
        month = np.repeat(np.arange(1, 13), dpm)
        day = np.concatenate([np.arange(1, n + 1) for n in dpm])
    return month, day, np.arange(1, month.size + 1)


def parse_offset(freq: str):
    """Mirror of ``xclim.core.calendar.parse_offset`` (core/calendar.py:558-606) for the frequencies
    the hot path uses: returns ``(multiplier, base, is_start_anchored, anchor)``."""
    m = re.fullmatch(r"(\d*)([A-Za-z]+?)(S|E)?(?:-([A-Za-z]{3}))?", freq)
    if not m:
        raise ValueError(f"Cannot parse frequency {freq!r}")
    mult, base, se, anchor = m.groups()
    mult = int(mult) if mult else 1
    base = base.upper()
    if base == "A":
        base = "Y"
    if base in ("Y", "Q", "M"):
        start = se == "S"
    else:
        start = True
    if anchor is not None:
        anchor = anchor.upper()
        if anchor not in _MONTHS:
            raise ValueError(f"Unknown anchor {anchor!r} in {freq!r}")
    elif base == "Y":
        anchor = "JAN" if start else "DEC"
    elif base == "Q":
        anchor = "JAN" if start else "DEC"  # pandas: QS == QS-JAN, QE == QE-DEC
    return mult, base, start, anchor


@dataclass
class TimeAxis:
    """A sorted, gap-free *daily* time axis described by its integer date fields."""

    year: np.ndarray
    month: np.ndarray
    day: np.ndarray
    doy: np.ndarray
    calendar: str = "standard"
    coord: object = None          # the original xarray time coordinate, when there was one
    _cache: dict = field(default_factory=dict, repr=False)

    # ------------------------------------------------------------------ constructors
    @classmethod
    def daily(cls, start: str, periods: int, calendar: str = "standard") -> "TimeAxis":
        """``periods`` consecutive days from ``start`` ("YYYY-MM-DD") in a CF ``calendar``."""
        if calendar not in MAX_DOY:
            raise ValueError(f"Unknown calendar {calendar!r}")
        y0, m0, d0 = (int(v) for v in start.split("-"))
        ys, ms, ds, js = [], [], [], []
        y = y0
        # offset of the start date inside its year
        mm, dd, jj = _year_fields(y, calendar)
        sel = np.nonzero((mm == m0) & (dd == d0))[0]
        if sel.size == 0:
            raise ValueError(f"{start} is not a valid date in calendar {calendar}")
        off = int(sel[0])
        need = periods
        while need > 0:
            mm, dd, jj = _year_fields(y, calendar)
            take = slice(off, min(mm.size, off + need))
            n = take.stop - take.start
            ys.append(np.full(n, y))
            ms.append(mm[take]); ds.append(dd[take]); js.append(jj[take])
            need -= n
            off = 0
            y += 1
        cat = lambda parts: np.concatenate(parts).astype(np.int32) if parts else np.zeros(0, np.int32)  # noqa: E731
        return cls(cat(ys), cat(ms), cat(ds), cat(js), calendar)

    @classmethod
    def from_xarray(cls, time) -> "TimeAxis":
        """From an xarray time coordinate (numpy datetime64 or cftime), via ``.dt``."""
        dt = time.dt
        cal = getattr(dt, "calendar", "standard")
        return cls(np.asarray(dt.year.values, np.int32), np.asarray(dt.month.values, np.int32),
                   np.asarray(dt.day.values, np.int32), np.asarray(dt.dayofyear.values, np.int32),
                   str(cal), coord=time)

    # ------------------------------------------------------------------ basic fields
    def __len__(self) -> int:
        return int(self.year.size)

    @property
    def max_doy(self) -> int:
        return MAX_DOY.get(self.calendar, 366)

    def isel(self, sl: slice) -> "TimeAxis":
        c = self.coord[sl] if self.coord is not None else None
        return TimeAxis(self.year[sl], self.month[sl], self.day[sl], self.doy[sl], self.calendar, coord=c)

    def sel_years(self, first: int, last: int) -> slice:
        """Index slice of the days whose calendar year is in ``[first, last]``
        (``da.sel(time=slice("first", "last"))`` with year-resolution strings)."""
        idx = np.nonzero((self.year >= first) & (self.year <= last))[0]
        if idx.size == 0:
            return slice(0, 0)
        return slice(int(idx[0]), int(idx[-1]) + 1)

    def sel_dates(self, first: str, last: str) -> slice:
        """``time.sel(time=slice(first, last))`` for "YYYY-MM-DD" bounds (both inclusive), as an index slice."""
        key = self.year.astype(np.int64) * 10000 + self.month * 100 + self.day
        f = int(first[:4]) * 10000 + int(first[5:7]) * 100 + int(first[8:10])
        la = int(last[:4]) * 10000 + int(last[5:7]) * 100 + int(last[8:10])
        return slice(int(np.searchsorted(key, f, side="left")), int(np.searchsorted(key, la, side="right")))

    def date_strings(self, idx) -> list[str]:
        idx = np.atleast_1d(idx)
        return [f"{int(self.year[i]):04d}-{int(self.month[i]):02d}-{int(self.day[i]):02d}" for i in idx]

    # ------------------------------------------------------------------ resampling
    def group_ids(self, freq: str) -> np.ndarray:
        """Monotonic integer id of the ``resample(time=freq)`` bin each day falls in."""
        mult, base, start, anchor = parse_offset(freq)
        y = self.year.astype(np.int64)
        m0 = self.month.astype(np.int64) - 1
        if base == "Y":
            am = _MONTHS.index(anchor)
            first_month = am if start else (am + 1) % 12
            gid = np.where(m0 >= first_month, y, y - 1)
        elif base == "Q":
            am = _MONTHS.index(anchor)
            first_month = (am if start else (am + 1)) % 3
            mon = y * 12 + m0 - first_month
            gid = np.floor_divide(mon, 3)
        elif base == "M":
            gid = y * 12 + m0
        elif base == "D":
            gid = np.arange(len(self), dtype=np.int64)
        else:
            raise NotImplementedError(f"frequency {freq!r} is not supported by the xclim_b200 hot path")
        if mult != 1:
            gid = np.floor_divide(gid - gid[0], mult) if gid.size else gid
        return gid

    def period_offsets(self, freq: str) -> np.ndarray:
        """int32 array of P+1 boundaries: period p covers ``[off[p], off[p+1])``.  ``freq=None`` is the
        reference's "no resampling" (indices/run_length.py:275-335 default): one period, the whole series."""
        if freq is None:
            return np.array([0, len(self)], dtype=np.int32)
        key = ("poff", freq)
        if key not in self._cache:
            gid = self.group_ids(freq)
            if gid.size == 0:
                off = np.zeros(1, np.int32)
            else:
                cuts = np.nonzero(np.diff(gid) != 0)[0] + 1
                off = np.concatenate([[0], cuts, [gid.size]]).astype(np.int32)
            self._cache[key] = off
        return self._cache[key]

    def period_labels(self, freq: str) -> list[str]:
        """Date label of every period as xarray would give it (period start for ``*S`` offsets,
        period end for ``*E``), as ISO strings."""
        mult, base, start, anchor = parse_offset(freq)
        off = self.period_offsets(freq)
        labels = []
        for p in range(off.size - 1):
            i = int(off[p])
            y, m = int(self.year[i]), int(self.month[i])
            if base == "D":
                labels.append(self.date_strings(i)[0])
                continue
            if base == "M":
                span = 1
                ms = m
                ys = y
            elif base == "Q":
                am = _MONTHS.index(anchor)
                first_month = (am if start else (am + 1)) % 3
                k = (y * 12 + m - 1 - first_month) // 3
                tot = k * 3 + first_month
                ys, ms = divmod(tot, 12)
                ms += 1
                span = 3
            else:
                am = _MONTHS.index(anchor)
                first_month = am if start else (am + 1) % 12
                ys = y if (m - 1) >= first_month else y - 1
                ms = first_month + 1
                span = 12
            if start:
                labels.append(f"{ys:04d}-{ms:02d}-01")
            else:
                tot = ys * 12 + ms - 1 + span * mult - 1
                ye, me = divmod(tot, 12)
                me += 1
                if self.calendar == "360_day":
                    dl = 30
                else:
                    dpm = _DPM_LEAP if bool(_is_leap(np.array(ye), self.calendar)) else _DPM_NOLEAP
                    dl = int(dpm[me - 1])
                labels.append(f"{ye:04d}-{me:02d}-{dl:02d}")
        return labels

    def _period_first_month(self, freq: str, p: int):
        """(year, month) of the first month of period ``p`` of ``resample(time=freq)`` and its span in months."""
        mult, base, start, anchor = parse_offset(freq)
        i = int(self.period_offsets(freq)[p])
        y, m = int(self.year[i]), int(self.month[i])
        if base == "M":
            return y, m, mult
        if base == "Q":
            am = _MONTHS.index(anchor)
            first_month = (am if start else (am + 1)) % 3
            tot = ((y * 12 + m - 1 - first_month) // 3) * 3 + first_month
            ys, ms = divmod(tot, 12)
            return ys, ms + 1, 3 * mult
        am = _MONTHS.index(anchor)
        first_month = am if start else (am + 1) % 12
        return (y if (m - 1) >= first_month else y - 1), first_month + 1, 12 * mult

    def _month_days(self, year: int, month0: int) -> int:
        if self.calendar == "360_day":
            return 30
        dpm = _DPM_LEAP if bool(_is_leap(np.array(year), self.calendar)) else _DPM_NOLEAP
        return int(dpm[month0])

    def expected_period_lengths(self, freq: str, **indexer) -> np.ndarray:
        """Number of daily steps every ``resample(time=freq)`` period holds in this calendar when it is
        complete -- ``expected_count`` of core/missing.py:64-160 for a daily source (``end_time -
        start_time`` between consecutive period labels).  A first / last period that the series only
        partly covers therefore expects more steps than it has.  With a ``select_time`` indexer (season,
        month, doy_bounds, date_bounds): the number of SELECTED days of the complete period (:122-141)."""
        mult, base, start, anchor = parse_offset(freq)
        P = self.period_offsets(freq).size - 1
        if base == "D":
            full = np.full(P, mult, np.int64)
            if not indexer:
                return full
            return np.add.reduceat(self.select_mask(**indexer).astype(np.int64), self.period_offsets(freq)[:-1])
        out = np.zeros(P, np.int64)
        for p in range(P):
            ys, ms, span = self._period_first_month(freq, p)
            n = 0
            for k in range(span):
                yy, mm = divmod(ys * 12 + ms - 1 + k, 12)
                n += self._month_days(yy, mm)
            out[p] = n
        if not indexer or P == 0:
            return out
        # a synthetic gap-free axis over the complete periods, select_time on it, count per period
        ys, ms, _ = self._period_first_month(freq, 0)
        full_axis = TimeAxis.daily(f"{ys:04d}-{ms:02d}-01", int(out.sum()), self.calendar)
        keep = full_axis.select_mask(**indexer).astype(np.int64)
        starts = np.concatenate([[0], np.cumsum(out)[:-1]])
        return np.add.reduceat(keep, starts)

    @staticmethod
    def bootstrap_freq(freq: str) -> str:
        """Year grouping used by the percentile bootstrap (core/bootstrapping.py:214-223):
        ``Y`` + ``S``/``E`` + the anchor of ``freq`` when its base is yearly or quarterly."""
        mult, base, start, anchor = parse_offset(freq)
        bfreq = "YS" if start else "YE"
        if base in ("Y", "Q") and anchor is not None:
            bfreq = f"{bfreq}-{anchor}"
        return bfreq

    def bootstrap_group_ids(self, freq: str) -> np.ndarray:
        """Group ids of the bootstrap year grouping of ``freq`` (``bootstrap_freq``)."""
        return self.group_ids(self.bootstrap_freq(freq))

    def date_index_in_periods(self, freq: str, date: str) -> np.ndarray:
        """Absolute index of the ``MM-DD`` date inside every ``resample(time=freq)`` group, -1 where the
        date is absent (``run_length.index_of_date`` per group, indices/run_length.py:1621-1665;
        more than one match in a group raises like the reference, :1663-1664)."""
        mm, dd = (int(v) for v in date.split("-"))
        off = self.period_offsets(freq)
        hit = np.nonzero((self.month == mm) & (self.day == dd))[0]
        out = np.full(off.size - 1, -1, np.int32)
        which = np.searchsorted(off, hit, side="right") - 1
        for p, t in zip(which, hit):
            if out[p] >= 0:
                raise ValueError(f"More than 1 instance of date {date} found in the coordinate array.")
            out[p] = t
        return out

    # ------------------------------------------------------------------ select_time
    def select_mask(self, season=None, month=None, doy_bounds=None, date_bounds=None, include_bounds=True):
        """Boolean step mask of ``select_time`` (core/calendar.py:1259-1376): exactly one of
        ``season`` ("DJF", ...), ``month``, ``doy_bounds`` (ints) or ``date_bounds`` ("MM-DD", "MM-DD")."""
        given = sum(a is not None for a in (season, month, doy_bounds, date_bounds))
        if given > 1:
            raise ValueError(f"Only one method of indexing may be given, got {given}.")
        if given == 0:
            return np.ones(len(self), bool)
        if isinstance(include_bounds, bool):
            include_bounds = (include_bounds, include_bounds)
        if season is not None:
            seasons = [season] if isinstance(season, str) else list(season)
            names = np.array(["DJF", "DJF", "MAM", "MAM", "MAM", "JJA", "JJA", "JJA", "SON", "SON", "SON", "DJF"])
            return np.isin(names[self.month - 1], seasons)
        if month is not None:
            months = [month] if isinstance(month, int) else list(month)
            return np.isin(self.month, months)
        if doy_bounds is not None:
            lo, hi = (int(v) for v in doy_bounds)
            return _between_doys(self.doy, lo, hi, include_bounds)
        start, end = date_bounds
        if self.calendar in ("noleap", "365_day", "360_day", "all_leap", "366_day"):
            cal, doy = self.calendar, self.doy
        else:  # non-uniform calendars are compared on the all_leap day numbers (:1343-1349)
            cal = "all_leap"
            doy = np.concatenate([[0], np.cumsum(_DPM_LEAP)])[self.month - 1] + self.day
        def dnum(md):
            mm, dd = (int(v) for v in md.split("-"))
            if cal == "360_day":
                return (mm - 1) * 30 + dd
            dpm = _DPM_LEAP if cal in ("all_leap", "366_day") else _DPM_NOLEAP
            return int(np.concatenate([[0], np.cumsum(dpm)])[mm - 1] + dd)
        return _between_doys(doy, dnum(start), dnum(end), include_bounds)


def _between_doys(doy, start, end, inclusive):
    """Steps whose day number lies between ``start`` and ``end`` (the interval wraps the year end when
    end < start); a bound flagged non-inclusive is excluded.  Same set as ``isin(_get_doys(...))`` of
    the reference (core/calendar.py:1137-1163)."""
    doy = np.asarray(doy)
    lo_ok = (doy >= start) if inclusive[0] else (doy > start)
    hi_ok = (doy <= end) if inclusive[1] else (doy < end)
    return (lo_ok & hi_ok) if start <= end else (lo_ok | hi_ok)
