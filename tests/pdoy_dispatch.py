"""Which kernels `xc_percentile_doy_f32` launches for a call: a restatement of `percentile_doy_impl`
(csrc/percentile_doy.cu) and of its launchers' day splits, so that each GPU test case can assert the kernel
it is meant to reach.  `plan_quantile` is the restatement shared with the bootstrap dispatch."""
import numpy as np

from boot_dispatch import plan_quantile

K_THREADS = 128          # cells per CTA of the generic, day-list and TMA kernels
K_SEL_THREADS = 64       # cells per CTA of the selection kernel
SEL_MAX_SAMPLES = 768    # samples per cell the selection kernel holds in shared memory
FAST_SMEM_CAP = 200 * 1024

# every template instance the dispatch can pick, named as the launches name them
INSTANCES = (
    [f"generic<{k}>" for k in (4, 8, 16, 32, 64)] + ["select"]
    + [f"uniform<{k}, {t}>" for k in (8, 16, 32) for t in ("false", "true")]
    + [f"w5p<{k}, {t}>" for k in (8, 16) for t in ("false", "true")]
    + [f"w5t<{n2}>" for n2 in (14, 15, 16)]
)


class Unsupported(Exception):
    """The call returns XC_ERR_UNSUPPORTED (NotImplementedError in Python)."""


def split_days(nd, cblocks, ctas_per_sm, min_per, pairs, sms):
    """common.cuh split_days: (chunks, days per chunk) of a launch over ``nd`` days and ``cblocks`` cell blocks."""
    chunks = max(1, (sms * ctas_per_sm + cblocks - 1) // cblocks)
    per = (nd + chunks - 1) // chunks
    per = max(per, min_per)
    if pairs:
        per = (per + 1) & ~1
    per = min(per, nd)
    return (nd + per - 1) // per, per


def _cblocks(C, threads=K_THREADS):
    return (C + threads - 1) // threads


class Launch:
    """One kernel launch: instance name, percentile index, day range [a, b) and its (chunks, per) day split."""

    def __init__(self, kernel, ip, a, b, split):
        self.kernel, self.ip, self.a, self.b = kernel, ip, a, b
        self.chunks, self.per = split

    @property
    def last_chunk(self):
        return (self.b - self.a) - (self.chunks - 1) * self.per

    def __repr__(self):
        return f"Launch({self.kernel!r}, p{self.ip}, [{self.a}, {self.b}), {self.chunks}x{self.per})"


def _generic(need, ip, a, b, C, sms):
    k = next(k for k in (4, 8, 16, 32, 64) if need <= k)
    return Launch(f"generic<{k}>", ip, a, b, split_days(b - a, _cblocks(C), 8, 1, False, sms))


def _day_lists(need, W, ip, a, b, C, table, sms):
    """launch_day_lists: the paired window-5 kernel for need <= 16, else the ring kernel."""
    t = "true" if table else "false"
    if W == 5 and need <= 16:
        k = 8 if need <= 8 else 16
        return Launch(f"w5p<{k}, {t}>", ip, a, b, split_days(b - a, _cblocks(C), 16, 40, True, sms))
    k = 8 if need <= 8 else 16 if need <= 16 else 32
    return Launch(f"uniform<{k}, {t}>", ip, a, b, split_days(b - a, _cblocks(C), 12, 8 * W, False, sms))


def kernel_plan(doy, year, n_doy, n_years, window, pers, C, ldx=None, aligned16=True, alpha=1 / 3, beta=1 / 3,
                no_tma=False, sms=132):
    """The launches of ``xc_percentile_doy_f32`` for a series with day-of-year ``doy`` (1-based) and year
    ordinal ``year`` per step, ``C`` cells in rows of ``ldx`` floats (default C) starting at a base pointer
    that is (``aligned16``) or is not 16-byte aligned.  ``no_tma``: XCLIM_B200_NO_TMA is set.  ``sms``: the
    device's multiprocessor count (the day splits depend on it).  Raises Unsupported where the call does."""
    doy = np.asarray(doy, dtype=np.int64)
    year = np.asarray(year, dtype=np.int64)
    T = doy.size
    ldx = C if ldx is None else ldx
    if window % 2 == 0:
        raise Unsupported("even window")
    h = window // 2
    pos = np.full((n_years, n_doy), -1, dtype=np.int64)
    pos[year, doy - 1] = np.arange(T)
    uniform = T == pos.size and bool((pos.ravel() == np.arange(pos.size)).all())
    L_int = 365 if n_doy == 366 else n_doy
    launches = []
    for ip, per in enumerate(np.atleast_1d(pers)):
        need, _ = plan_quantile(float(per), alpha, beta, n_years * window)
        if need < 0:
            raise Unsupported("plotting positions outside [0, 1]")
        if need > 64:
            if n_years * window > SEL_MAX_SAMPLES:
                raise Unsupported("more samples than the selection kernel holds")
            launches.append(Launch("select", ip, 0, n_doy, split_days(n_doy, _cblocks(C, K_SEL_THREADS), 8, 1,
                                                                      False, sms)))
            continue
        kk = 8 if need <= 8 else 16 if need <= 16 else 32
        smem = (window - 1) * (kk + 1) * K_THREADS * 4
        fast_ok = window >= 3 and need <= 32 and smem <= FAST_SMEM_CAP and L_int - 2 * h >= 8
        if uniform and fast_ok:
            tma = (window == 5 and 8 < need <= 16 and not no_tma and 30 <= n_years <= 32 and ldx % 4 == 0
                   and aligned16 and n_doy >= 8)
            if tma:
                split = split_days(n_doy, _cblocks(C), 12, 40, True, sms)
                launches.append(Launch(f"w5t<{n_years - 16}>", ip, 0, n_doy, split))
            else:
                launches.append(_day_lists(need, window, ip, 0, n_doy, C, False, sms))
            continue
        # table mode: per-day lists on the days whose windows stay inside the year and around no missing
        # centre (the h days before the first step's day-of-year and after the last step's), generic elsewhere
        fast_day = np.zeros(n_doy, dtype=bool)
        if fast_ok:
            fast_day[h:L_int - h] = True
            s0, e1 = int(doy[0]) - 1, int(doy[-1]) - 1
            fast_day[max(0, s0 - h):s0] = False
            fast_day[e1 + 1:e1 + 1 + h] = False
        a = 0
        while a < n_doy:
            b = a
            while b < n_doy and fast_day[b] == fast_day[a]:
                b += 1
            if fast_day[a] and b - a >= 8:
                launches.append(_day_lists(need, window, ip, a, b, C, True, sms))
            else:
                launches.append(_generic(need, ip, a, b, C, sms))
            a = b
    return launches


def kernels(*args, **kw):
    """The set of instance names ``kernel_plan`` launches."""
    return {ln.kernel for ln in kernel_plan(*args, **kw)}


def uniform_calendar(L, n_years):
    """(doy, year) of ``n_years`` whole years of ``L`` days."""
    t = np.arange(L * n_years)
    return t % L + 1, t // L
