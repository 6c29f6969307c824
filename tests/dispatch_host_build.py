"""TEST INFRASTRUCTURE: build and bind the host build of the launch plans (tests/csrc/dispatch_host.cu over
xclim_b200/csrc/launch_plan.cuh), so that a test names the kernel instance a call runs by asking the launchers' own
dispatch.  Calls the library rejects raise Unsupported (XC_ERR_UNSUPPORTED) or ValueError."""
import ctypes

import numpy as np

import host_build
from xclim_b200 import _lib as L

_vp, _i64, _i32, _f64 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_double
SIGNATURES = {
    "dispatch_error": (ctypes.c_char_p, []),
    "dispatch_name": (ctypes.c_char_p, [_i32, _i32]),
    "dispatch_split_days": (None, [_i32, _i64, _i32, _i32, _i32, _i32, _i32, _vp]),
    "dispatch_plan_quantile": (_i32, [_f64, _f64, _f64, _i32, _vp]),
    "dispatch_pdoy": (_i32, [_i64, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _i32, _f64, _f64, _i64, _i64, _i32, _i32,
                             _i32, _vp, _i32, _vp]),
    "dispatch_boot_exact_above": (_i32, []),
    "dispatch_bootstrap": (_i32, [_i32, _i32, _i32, _f64, _f64, _f64, _i32, _i32, _i64, _i32, _vp]),
    "dispatch_can_stream4": (_i32, [_i64, _i64, _i32, _i32, _i32]),
    "dispatch_roll_slides": (_i32, [_i32, _i32, _i32]),
    "dispatch_rolling": (_i32, [_i64, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _i32]),
    "dispatch_multi_check": (_i32, [_vp, _i32]),
    "dispatch_multi_shape": (None, [_i32, _i32, _i32, _i32, _vp]),
}
H100_SMS = 132


class Unsupported(NotImplementedError):
    """The call returns XC_ERR_UNSUPPORTED (NotImplementedError in Python)."""


def load():
    return host_build.load("dispatch", "dispatch_host.cu", nvcc=True, signatures=SIGNATURES)


def _check(status):
    if status:
        msg = load().dispatch_error().decode()
        raise Unsupported(msg) if status == L.XC_ERR_UNSUPPORTED else ValueError(msg)


def _names(table):
    names = []
    while name := load().dispatch_name(table, len(names)).decode():
        names.append(name)
    return names


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def split_plan(nd, cblocks, ctas_per_sm, min_per, pairs, sms=H100_SMS, align=1):
    """(chunks, days per chunk) of a day-of-year launch over ``nd`` days and ``cblocks`` cell blocks."""
    out = np.zeros(2, np.int32)
    load().dispatch_split_days(nd, cblocks, ctas_per_sm, min_per, int(pairs), align, sms, _p(out))
    return int(out[0]), int(out[1])


def quantile_plan(per, alpha, beta, n_max):
    """(need, top): the order statistics kept on the chosen side of samples of up to ``n_max`` values and whether
    that side is the top (largest values); need = -1 when neither side works."""
    top = ctypes.c_int32(0)
    return load().dispatch_plan_quantile(per, alpha, beta, n_max, ctypes.byref(top)), bool(top.value)


# ---- percentile_doy
PDOY_INSTANCES = _names(0)


class Launch:
    """One kernel launch: instance name, percentile index, day range [a, b), its (chunks, per) day split and its
    dynamic shared memory."""

    def __init__(self, kernel, ip, a, b, chunks, per, smem):
        self.kernel, self.ip, self.a, self.b, self.chunks, self.per, self.smem = \
            PDOY_INSTANCES[kernel], ip, a, b, chunks, per, smem

    @property
    def last_chunk(self):
        return (self.b - self.a) - (self.chunks - 1) * self.per

    def __repr__(self):
        return f"Launch({self.kernel!r}, p{self.ip}, [{self.a}, {self.b}), {self.chunks}x{self.per})"


def pdoy_plan(doy, year, n_doy, n_years, window, pers, C, ldx=None, aligned16=True, alpha=1 / 3, beta=1 / 3,
              no_tma=False, sms=H100_SMS, has_vrow=False):
    """The launches of ``xc_percentile_doy_f32`` (``has_vrow``: ``_vrow_f32``) for a series with day-of-year ``doy``
    (1-based) and year ordinal ``year`` per step, ``C`` cells in rows of ``ldx`` floats (default C) from a base
    pointer that is (``aligned16``) or is not 16-byte aligned.  ``no_tma``: XCLIM_B200_NO_TMA is set; ``sms``: the
    device's multiprocessor count (the day splits depend on it)."""
    doy, year = np.ascontiguousarray(doy, dtype=np.int16), np.ascontiguousarray(year, dtype=np.int16)
    pers = np.ascontiguousarray(np.atleast_1d(pers), dtype=np.float64)
    cap, n = 8 * n_doy * pers.size, ctypes.c_int32(0)
    out = np.zeros((cap, 7), np.int64)
    _check(load().dispatch_pdoy(doy.size, _p(doy), _p(year), int(has_vrow), n_doy, n_years, window, _p(pers),
                                pers.size, alpha, beta, C, C if ldx is None else ldx, int(aligned16), int(no_tma),
                                sms, _p(out), cap, ctypes.byref(n)))
    assert n.value <= cap
    return [Launch(*(int(v) for v in row)) for row in out[:n.value]]


def pdoy_kernels(*args, **kw):
    """The set of instance names ``pdoy_plan`` launches."""
    return {ln.kernel for ln in pdoy_plan(*args, **kw)}


# ---- bootstrap
BOOT_KERNELS = _names(1)


def boot_plan(n_base_years, window, per, alpha=1 / 3, beta=1 / 3, year_len=365, boot_v1=False, mask=False, C=1,
              sms=H100_SMS):
    """(kernel, chunks, days per chunk, shared memory) of the bootstrap's exceedance launch: kernel 'bootstrap5',
    '16x8', '32x16' or '32x32' (bootstrap_kernel<KA, KB>).  ``mask``: the per-pair masks of
    xc_bootstrap_doy_index_f32; ``boot_v1``: XCLIM_B200_BOOT_V1 is set."""
    out = np.zeros(4, np.int64)
    _check(load().dispatch_bootstrap(n_base_years, year_len, window, per, alpha, beta, int(mask), int(boot_v1), C,
                                     sms, _p(out)))
    return BOOT_KERNELS[out[0]], int(out[1]), int(out[2]), int(out[3])


def boot_kernel(n_base_years, window, per, alpha=1 / 3, beta=1 / 3, year_len=365, boot_v1=False):
    """The kernel name of ``boot_plan``, or None where the call raises NotImplementedError."""
    try:
        return boot_plan(n_base_years, window, per, alpha, beta, year_len, boot_v1)[0]
    except Unsupported:
        return None


def exact_years(n_base_years):
    """bootstrap_kernel skips its rank shortcuts (every year takes the exact per-(y, s) loop)."""
    return n_base_years > load().dispatch_boot_exact_above()


# ---- rolling windows and spells
SUM, MEAN, MIN, MAX = (L.STATS[k] for k in ("sum", "mean", "min", "max"))
_FAMILIES = {name: f for f, name in enumerate(_names(2))}

# the instantiated kernels: spell_sumw<W, RED, AFTER> and rolling_sumw<W, MODE> for the register windows 2..8,
# RED one of XC_RL_MAX / SUM / COUNT or kRunAny (-1), MODE 0 max / 1 min / 2 the other statistics
SPELL_SUMW = [f"spell_sumw<{w}, {red}, {after}>" for w in range(2, 9) for red in (0, 2, 3, -1)
              for after in ("false", "true")]
ROLLING_SUMW = [f"rolling_sumw<{w}, {mode}>" for w in range(2, 9) for mode in (0, 1, 2)]
INSTANCES = SPELL_SUMW + ROLLING_SUMW + ["spell_runstat4<false>", "spell_runstat4<true>", "rolling_period_reduce4",
                                         "spell_runstat", "rolling_period_reduce", "spell_mask"]
#: the instances that keep a running float64 sum for some sum / mean windows
SLIDING = {"rolling_period_reduce4", "spell_runstat4<false>", "spell_runstat4<true>", "rolling_period_reduce",
           "spell_runstat", "spell_mask"}


def can_stream4(C, ldx, window, aligned_x=True, aligned_out=True):
    """4 cells per thread need 16-byte rows and a ring that fits shared memory."""
    return bool(load().dispatch_can_stream4(C, ldx, int(aligned_x), int(aligned_out), window))


def instance_slides(kernel, window, wstat):
    """Whether ``kernel`` keeps a running window sum (new value in, oldest out) for this window."""
    return bool(load().dispatch_roll_slides(_FAMILIES[kernel.split("<")[0]], window, wstat))


def _roll(C, ldx, window, wstat, center, stat, before, aligned_x):
    name = ctypes.create_string_buffer(64)
    _check(load().dispatch_rolling(C, ldx, int(aligned_x), window, wstat, center, stat, int(before), name, 64))
    return name.value.decode()


def spell_instance(C, ldx, window, wstat, reducer, resample_before_rl=True, aligned_x=True):
    """The instance ``xc_spell_runstat_f32`` launches; ``reducer`` is the run-length reducer code."""
    return _roll(C, ldx, window, wstat, -1, reducer, resample_before_rl, aligned_x)


def rolling_instance(C, ldx, window, wstat, stat, center=False, aligned_x=True):
    """The instance ``xc_rolling_period_reduce_f32`` launches; ``stat`` is the per-period statistic code."""
    return _roll(C, ldx, window, wstat, int(center), stat, True, aligned_x)


# ---- the fused multi-output pass
def multi_errors(plan, n_slots):
    """The error of `xc_period_multi_f32` on ``plan`` as a list (empty: accepted), output buffers aside."""
    st = load().dispatch_multi_check(ctypes.byref(type(plan).from_buffer_copy(plan)), n_slots)
    return [load().dispatch_error().decode()] if st else []


def multi_shape(plan):
    """(NC, NCR, NM, NS, VEC, UNROLL) of the period_multi_kernel instantiation that runs ``plan``."""
    out = np.zeros(6, np.int32)
    load().dispatch_multi_shape(plan.n_cond, plan.n_runs, plan.n_msum, plan.n_sums, _p(out))
    return tuple(int(v) for v in out)
