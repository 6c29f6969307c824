"""The fused multi-output pass seen from the host: a restatement of the plan checks and of the dispatch of
`xc_period_multi_f32` (csrc/period_stats.cu), so that a test can assert that a plan is accepted and name the
`period_multi_kernel<NC, NCR, NM, NS, VEC, UNROLL>` instantiation it runs."""
from xclim_b200 import _lib

MAX_COND, MAX_RUNS, MAX_MSUM, MAX_SUMS = _lib.MULTI_MAX_COND, _lib.MULTI_MAX_RUNS, _lib.MULTI_MAX_MSUM, \
    _lib.MULTI_MAX_SUMS


def plan_errors(plan, n_slots):
    """The reasons `xc_period_multi_f32` rejects ``plan`` (empty: accepted), buffer checks aside."""
    errs = []
    if not (0 <= plan.n_cond <= MAX_COND and 0 <= plan.n_runs <= MAX_RUNS and plan.n_runs % 2 == 0 and
            0 <= plan.n_msum <= MAX_MSUM and 0 <= plan.n_sums <= MAX_SUMS):
        errs.append("counts")
    if plan.n_runs // 2 > plan.n_cond or (plan.n_msum and plan.n_cond == 0):
        errs.append("run outputs need their condition")

    def slot_ok(s):
        return -1 <= s < n_slots
    ok = all(slot_ok(s) for s in (plan.slot_sum, plan.slot_mean, plan.slot_min, plan.slot_max))
    for j in range(min(plan.n_cond, MAX_COND)):
        ok = ok and slot_ok(plan.cond[j].slot_n) and slot_ok(plan.cond[j].slot_max)
    for k in range(min(plan.n_runs, MAX_RUNS)):
        r = plan.runs[k]
        ok = ok and slot_ok(r.slot) and r.window >= 1 and r.kind in (0, 1) and r.cond == k // 2
    for k in range(min(plan.n_msum, MAX_MSUM)):
        m = plan.msum[k]
        ok = ok and slot_ok(m.slot) and m.window >= 1 and m.cond == 0
    for k in range(min(plan.n_sums, MAX_SUMS)):
        ok = ok and slot_ok(plan.sums[k].slot) and plan.sums[k].mode in (0, 1)
    if not ok:
        errs.append("slots / windows / run places")
    return errs


def multi_kernel(plan):
    """(NC, NCR, NM, NS, VEC, UNROLL) of the instantiation that runs ``plan``: the counts rounded up to the
    instantiated shapes; four cells per thread only for passes without run outputs, run sums or conditional sums
    and with at most two conditions."""
    nc = 0 if plan.n_cond == 0 else (2 if plan.n_cond <= 2 else (4 if plan.n_cond <= 4 else 6))
    ncr, nm, ns = plan.n_runs // 2, plan.n_msum, 0 if plan.n_sums == 0 else 3
    vec, unroll = (4, 8) if (ncr == 0 and nm == 0 and ns == 0 and nc <= 2) else (2, 12)
    return nc, ncr, nm, ns, vec, unroll


def instantiations():
    """The 38 instantiated (NC, NCR, NM, NS)."""
    out = [(0, 0, 0, 0), (0, 0, 0, 3)]
    for nc in (2, 4, 6):
        for nm in (0, 1):
            for ncr in (0, 1, 2):
                for ns in (0, 3):
                    out.append((nc, ncr, nm, ns))
    return out


def empty_plan():
    plan = _lib.MultiPlan()
    plan.slot_sum = plan.slot_mean = plan.slot_min = plan.slot_max = -1
    for j in range(MAX_COND):
        plan.cond[j].slot_n = plan.cond[j].slot_max = -1
        plan.cond[j].wmax = 1
    for k in range(MAX_RUNS):
        plan.runs[k].cond, plan.runs[k].window, plan.runs[k].slot = k // 2, 1, -1
    plan.msum[0].slot, plan.msum[0].window = -1, 1
    for k in range(MAX_SUMS):
        plan.sums[k].slot = -1
    return plan
