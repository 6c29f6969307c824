"""Which kernel `xc_bootstrap_doy_count_f32` runs for a given bootstrap: a restatement of
`plan_quantile` (csrc/quantile.cuh) and of the dispatch in csrc/bootstrap.cu, so that each test case can
assert the branch it is meant to exercise."""
import math


def plan_quantile(per, alpha, beta, n_max):
    """(need, top): the number of order statistics kept on the chosen side of samples of up to ``n_max``
    values, and whether that side is the top (largest values).  need = -1 when neither side works."""
    q = per / 100.0
    c = alpha + q * (1 - alpha - beta)
    ktop = kbot = 1
    for n in range(2, n_max + 1):
        vi = float(n) * q + c - 1
        if vi >= n - 1 or vi < 0:
            continue
        lo = int(math.floor(vi))
        ktop = max(ktop, n - lo)
        kbot = max(kbot, lo + 2)
    top_ok = bot_ok = True
    for n in range(2, n_max + 1):
        vi = float(n) * q + c - 1
        if vi < 0:
            top_ok = False
        if vi >= n - 1:
            bot_ok = False
    if top_ok and (ktop <= kbot or not bot_ok):
        return ktop, True
    if bot_ok:
        return kbot, False
    return -1, False


def bootstrap_kernel(n_base_years, window, per, alpha=1 / 3, beta=1 / 3, year_len=365, boot_v1=False):
    """'bootstrap5', '16x8', '32x16', '32x32' (bootstrap_kernel<KA, KB>) or None (NotImplementedError).
    ``boot_v1``: XCLIM_B200_BOOT_V1 is set (the general kernel even where bootstrap5 applies)."""
    need, _ = plan_quantile(per, alpha, beta, n_base_years * window)
    if (0 < need <= 8 and window == 5 and n_base_years <= 16 and year_len > 8 and not boot_v1):
        return "bootstrap5"
    if 0 < need <= 8 and need + window <= 16:
        return "16x8"
    if 0 < need <= 16 and need + window <= 32:
        return "32x16"
    if 0 < need and need + window <= 32:
        return "32x32"
    return None


def every_year_exact(n_base_years):
    """bootstrap_kernel skips its rank shortcuts (every year takes the exact per-(y, s) loop) above 32 years."""
    return n_base_years > 32
