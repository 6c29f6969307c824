"""Which kernel `xc_rolling_period_reduce_f32`, `xc_spell_runstat_f32` and `xc_spell_mask_f32` launch for a
call: a restatement of their dispatch (csrc/rolling.cu), so that each GPU test case can assert the kernel it
is meant to reach, and whether that kernel keeps a sliding float64 window sum (new value in, oldest out)
instead of summing every window afresh.  Instances are named as the launches name them."""
K_THREADS = 128
RING_SMEM_CAP = 160 * 1024    # shared memory the ring kernels may ask for: w * 128 threads * 16 bytes

SUM, MEAN, MIN, MAX = 0, 1, 2, 3                        # window statistics (_lib.STATS)
RL_MAX, RL_SUM, RL_COUNT, RUN_ANY = 0, 2, 3, -1         # spell_sumw_kernel's RED argument (runstat.cuh)
REGISTER_WINDOWS = range(2, 9)                          # XC_DISPATCH_W: the register kernels' W

SPELL_SUMW = [f"spell_sumw<{w}, {red}, {after}>" for w in REGISTER_WINDOWS for red in (RL_MAX, RL_SUM, RL_COUNT,
                                                                                      RUN_ANY)
              for after in ("false", "true")]
ROLLING_SUMW = [f"rolling_sumw<{w}, {mode}>" for w in REGISTER_WINDOWS for mode in (0, 1, 2)]
SPELL_RING = ["spell_runstat4<false>", "spell_runstat4<true>"]
ROLLING_RING = ["rolling_period_reduce4"]
LANE = ["spell_runstat", "rolling_period_reduce", "spell_mask"]
INSTANCES = SPELL_SUMW + ROLLING_SUMW + SPELL_RING + ROLLING_RING + LANE

#: kernels that keep a running float64 sum for sum / mean windows (spell_runstat and spell_mask only above
#: window 6, see BlockStream::sliding); the register kernels re-add each window from their registers
SLIDING = {"rolling_period_reduce4", "spell_runstat4<false>", "spell_runstat4<true>", "rolling_period_reduce",
           "spell_runstat", "spell_mask"}


class Unsupported(Exception):
    """The call returns XC_ERR_UNSUPPORTED (NotImplementedError in Python)."""


def can_stream4(C, ldx, window, aligned_x=True, aligned_out=True):
    """rolling.cu can_stream4: 4 cells per thread need 16-byte rows and a ring that fits shared memory."""
    return (C % 4 == 0 and ldx % 4 == 0 and aligned_x and aligned_out
            and window * K_THREADS * 16 <= RING_SMEM_CAP)


def _is_sum(wstat):
    return wstat in (SUM, MEAN)


def rolling_kernel(C, ldx, window, wstat, stat, center=False, aligned_x=True):
    """The instance ``xc_rolling_period_reduce_f32`` launches; ``stat`` is the per-period statistic code."""
    if center and window % 2 == 0:
        raise Unsupported("centred rolling windows of even length")
    s4 = can_stream4(C, ldx, window, aligned_x)
    if s4 and _is_sum(wstat) and window in REGISTER_WINDOWS:
        mode = 0 if stat == MAX else 1 if stat == MIN else 2
        return f"rolling_sumw<{window}, {mode}>"
    return "rolling_period_reduce4" if s4 else "rolling_period_reduce"


def spell_kernel(C, ldx, window, wstat, reducer, resample_before_rl=True, aligned_x=True):
    """The instance ``xc_spell_runstat_f32`` launches; ``reducer`` is the run-length reducer code."""
    after = "false" if resample_before_rl else "true"
    s4 = can_stream4(C, ldx, window, aligned_x)
    if s4 and _is_sum(wstat) and window in REGISTER_WINDOWS:
        red = reducer if reducer in (RL_MAX, RL_SUM, RL_COUNT) else RUN_ANY
        return f"spell_sumw<{window}, {red}, {after}>"
    return f"spell_runstat4<{after}>" if s4 else "spell_runstat"


def slides(kernel, window, wstat):
    """Whether ``kernel`` keeps a running window sum for this window."""
    if kernel not in SLIDING or not _is_sum(wstat):
        return False
    return window > 6 if kernel in ("spell_runstat", "spell_mask") else True
