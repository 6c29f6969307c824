"""Shared test helpers (imported as a top-level module: the tests directory is on sys.path)."""
import numpy as np


def make_field(values, start="2000-01-01", calendar="standard", units="K", dims=None, **attrs):
    """A Field with a daily time axis on dim 0 (the `*_series` fixtures of the reference's
    tests/conftest.py, without xarray)."""
    from xclim_b200 import Field, TimeAxis
    values = np.asarray(values)
    ta = TimeAxis.daily(start, values.shape[0], calendar)
    if dims is None:
        dims = ("time",) + tuple(f"d{i}" for i in range(values.ndim - 1))
    return Field(values, dims, ta, {}, {"units": units, **attrs})


def uniform_calendar(L, n_years):
    """(doy, year) of ``n_years`` whole years of ``L`` days."""
    t = np.arange(L * n_years)
    return t % L + 1, t // L


def instantiations():
    """The 38 instantiated (NC, NCR, NM, NS) of period_multi_kernel."""
    out = [(0, 0, 0, 0), (0, 0, 0, 3)]
    for nc in (2, 4, 6):
        for nm in (0, 1):
            for ncr in (0, 1, 2):
                for ns in (0, 3):
                    out.append((nc, ncr, nm, ns))
    return out


def empty_plan():
    """A fused-pass plan with no outputs: every slot -1, every entry at its neutral value."""
    from xclim_b200 import _lib
    plan = _lib.MultiPlan()
    plan.slot_sum = plan.slot_mean = plan.slot_min = plan.slot_max = -1
    for j in range(_lib.MULTI_MAX_COND):
        plan.cond[j].slot_n = plan.cond[j].slot_max = -1
        plan.cond[j].wmax = 1
    for k in range(_lib.MULTI_MAX_RUNS):
        plan.runs[k].cond, plan.runs[k].window, plan.runs[k].slot = k // 2, 1, -1
    plan.msum[0].slot, plan.msum[0].window = -1, 1
    for k in range(_lib.MULTI_MAX_SUMS):
        plan.sums[k].slot = -1
    return plan


def plant_infinite_samples(x, qs, cells, seed=0):
    """Overwrite five cells per quantile q of ``x`` (time first; ``cells`` are flat cell indexes, used in
    order) with infinite or overflowing values placed around the q-quantile's neighbours, so that the
    interpolation meets +inf at the top ranks, a -inf left neighbour, the pair {-inf, +inf} (also in
    two-value samples) and finite +-3e38 whose difference overflows float32.  Returns the cells used."""
    rng = np.random.default_rng(seed)
    flat = x.reshape(x.shape[0], -1)
    assert np.shares_memory(flat, x)
    T = x.shape[0]
    big = np.float32(3e38)
    used = []
    it = iter(cells)
    for q in qs:
        u = rng.random(T)
        c = next(it); flat[u < 1.1 * (1 - q), c] = np.inf; used.append(c)          # +inf at the top ranks
        c = next(it); flat[u < 1.1 * q, c] = -np.inf; used.append(c)               # -inf left neighbours
        c = next(it); flat[:, c] = np.where(u < q, -np.inf, np.inf); used.append(c)  # {-inf, +inf}
        v = np.where(rng.random(T) < 0.5, -np.inf, np.inf)
        c = next(it); flat[:, c] = np.where(rng.random(T) < 0.985, np.nan, v); used.append(c)
        c = next(it); used.append(c)                                                # +-3e38 and +inf next to -3e38
        flat[:, c] = np.where(u < 0.9 * q, -big, np.where(u > 1 - 0.9 * (1 - q), big, flat[:, c]))
        flat[(u > 0.5 * q) & (u < 0.5 * q + 0.05), c] = np.inf
    return used
