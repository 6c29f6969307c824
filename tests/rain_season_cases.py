"""TEST INFRASTRUCTURE: seeded rain-season cases shared by the CPU test of the host build and the GPU test of the
kernel.  Each case is a (T, C) float32 series on a daily time axis with one parameter set of `rain_season`.

The series alternate 10-day wet and dry regimes in quarter-mm amounts (so that window sums are exact), with the
thresholds and their float32 neighbours, NaN days and NaN runs, signed zeros and infinities sprinkled in, and a few
planted cells: an event run that qualifies on the last steps of a period, a dry tail that fills a whole `total` end
window, a start whose day is the period's last."""
import numpy as np

from xclim_b200.timeaxis import TimeAxis

START_BOUNDS = [("05-01", "12-31"), ("01-01", "12-31"), ("03-01", "06-30"), ("06-15", "06-15"), ("11-01", "02-28"),
                ("12-31", "01-01"), ("07-01", "12-31")]
END_BOUNDS = [("09-01", "12-31"), ("01-01", "12-31"), ("07-01", "07-01"), ("10-15", "03-31"), ("06-01", "12-31")]
AXES = [("noleap", "2000-01-01", 730), ("360_day", "1999-07-15", 800), ("all_leap", "2001-03-10", 1000),
        ("standard", "2000-01-01", 1096), ("standard", "1999-09-20", 470), ("noleap", "2000-05-20", 330)]


def neighbours(v):
    v = np.float32(v)
    return [v, np.nextafter(v, np.float32(np.inf)), np.nextafter(v, np.float32(-np.inf))]


def series(rng, T, C, params, scale):
    """(T, C) float32 rates whose amounts (times ``scale``) follow the regimes above."""
    wet_p = rng.uniform(0.2, 0.9, C)
    regime = rng.random((T // 10 + 1, C)) < wet_p
    wet = np.repeat(regime, 10, axis=0)[:T]
    amt = np.where(wet, rng.integers(0, 60, (T, C)) / 4.0,
                   np.where(rng.random((T, C)) < 0.8, 0.0, rng.integers(0, 5, (T, C)) / 4.0)).astype(np.float32)
    specials = [np.float32(-0.0), np.float32(np.inf), np.float32(-np.inf)]
    for k in ("thresh_wet_start", "thresh_dry_start", "thresh_dry_end"):
        specials += neighbours(params[k])
    specials += neighbours(np.float32(params["thresh_wet_start"]) / max(1, params["window_wet_start"]))
    hit = rng.random((T, C)) < 0.03
    amt[hit] = rng.choice(np.array(specials, np.float32), hit.sum())
    amt[rng.random((T, C)) < 0.01] = np.nan
    for c in rng.choice(C, max(1, C // 8), replace=False):       # NaN runs
        t = rng.integers(0, T)
        amt[t:t + rng.integers(2, 12), c] = np.nan
    return (amt / np.float32(scale)).astype(np.float32) if scale != 1.0 else amt


def plant(x, poff, params, scale, rng):
    """A few cells per period with a pattern on the period's edges (see the module doc)."""
    C = x.shape[1]
    N = params["window_not_dry_start"] + params["window_wet_start"]
    big = np.float32(params["thresh_wet_start"]) + 10
    for a, b in zip(poff[:-1], poff[1:]):
        n = b - a
        c = rng.integers(0, C, 4)
        if n > N + 2:                                     # the last event run that can still qualify
            x[b - N - 2:b, c[0]] = 0
            x[b - N:b, c[0]] = big / scale
        x[b - 1, c[1]] = big / scale                      # wet on the last day only
        x[b - 80 if n > 80 else a:b, c[2]] = 0            # a dry tail: every end window in it qualifies
        x[a:b, c[3]] = big / scale                        # all wet: no dry sequence anywhere


def cases(seed, dry_start_method, n_cases):
    """Yields ``(x, ta, freq, scale, params)``."""
    rng = np.random.default_rng(seed)
    for i in range(n_cases):
        cal, start, T = AXES[i % len(AXES)]
        ta = TimeAxis.daily(start, T, cal)
        freq = ("YS-JAN", "YS-JUL")[(i // len(AXES)) % 2]
        ds, de = START_BOUNDS[rng.integers(len(START_BOUNDS))], END_BOUNDS[rng.integers(len(END_BOUNDS))]
        params = dict(
            thresh_wet_start=float(rng.choice([25.0, 10.0, 5.25, 0.0])),
            window_wet_start=int(rng.choice([1, 2, 3, 4])),
            window_not_dry_start=int(rng.choice([0, 1, 3, 10, 30])),
            thresh_dry_start=float(rng.choice([1.0, 0.5, 0.0, 0.25])),
            window_dry_start=int(rng.choice([1, 2, 3, 7, 64])),
            method_dry_start=dry_start_method,
            date_min_start=ds[0], date_max_start=ds[1],
            thresh_dry_end=float(rng.choice([0.0, 0.25, 1.0, 2.0])),
            window_dry_end=int(rng.choice([1, 2, 5, 20, 64])),
            method_dry_end=("per_day", "total")[i % 2],
            date_min_end=de[0], date_max_end=de[1])
        scale = 86400.0 if i % 5 == 4 else 1.0
        x = series(rng, T, 256, params, scale)
        plant(x, ta.period_offsets(freq), params, np.float32(scale), rng)
        yield x, ta, freq, scale, params
