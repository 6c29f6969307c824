"""Sequential restatement of the fused multi-output pass (``xc_period_multi_f32``, ``XcMultiPlan`` in
include/xclim_b200.h): every output of a plan, computed the way the kernel computes it, so that each slot can be
compared bit for bit.

Per period and cell, in time order:
  * sum / mean / min / max of the non-NaN values, the sum accumulated in float64;
  * per condition ``sgn * x > thr`` (float32): the number of true steps and the longest run, reported as 0 when
    it is shorter than ``wmax``;
  * per run output k (condition k // 2): the total length (kind 0) or the number (kind 1) of the runs at least
    ``window`` long, the run that the period end closes included;
  * the largest float64 sum of the float32 excesses ``sgn * (x - thr0)`` over the runs of condition 0 at least
    ``window`` long (0 when there is none);
  * conditional sums in float64: mode 0 adds ``max(off_sgn * (x - off), 0)`` (float32) over the non-NaN steps,
    mode 1 adds ``x`` where ``sgn * x > thr``.
Only the declared entries (``n_cond``, ``n_runs``, ``n_msum``, ``n_sums``) are computed.  ``plan`` is any object
with the attributes of ``xclim_b200._lib.MultiPlan``; the float64 accumulators are summed one step after the
other, as the kernel does, never pairwise.
"""
import numpy as np

F32 = np.float32


def period_multi_raw(x, poff, plan):
    """{output: (P, C) array} before the final float32 rounding.  Keys: "sum", "mean", "min", "max",
    ("n", j), ("max", j), ("run", k), ("msum", 0), ("qsum", k); "n" and the run outputs are int64, the sums and
    the mean float64, min / max float32."""
    x = np.asarray(x, dtype=F32)
    poff = np.asarray(poff, dtype=np.int64)
    P, C = len(poff) - 1, x.shape[1]
    nc, nr, nm, ns = int(plan.n_cond), int(plan.n_runs), int(plan.n_msum), int(plan.n_sums)
    conds = [(F32(plan.cond[j].sgn), F32(plan.cond[j].thr), int(plan.cond[j].wmax)) for j in range(nc)]
    runs = [(k // 2, int(plan.runs[k].window), int(plan.runs[k].kind)) for k in range(nr)]
    sums = [(int(plan.sums[k].mode), F32(plan.sums[k].sgn), F32(plan.sums[k].thr), F32(plan.sums[k].off_sgn),
             F32(plan.sums[k].off)) for k in range(ns)]
    if nm:
        m_w, m_sgn, m_thr0 = int(plan.msum[0].window), F32(plan.msum[0].sgn), F32(plan.msum[0].thr0)
    res = {k: np.zeros((P, C), np.float64) for k in ("sum", "mean")}
    res["min"] = np.zeros((P, C), F32)
    res["max"] = np.zeros((P, C), F32)
    for j in range(nc):
        res[("n", j)] = np.zeros((P, C), np.int64)
        res[("max", j)] = np.zeros((P, C), np.int64)
    for k in range(nr):
        res[("run", k)] = np.zeros((P, C), np.int64)
    if nm:
        res[("msum", 0)] = np.zeros((P, C), np.float64)
    for k in range(ns):
        res[("qsum", k)] = np.zeros((P, C), np.float64)
    with np.errstate(all="ignore"):
        for p in range(P):
            s = np.zeros(C)
            nok = np.zeros(C, np.int64)
            mn = np.full(C, np.inf, F32)
            mx = np.full(C, -np.inf, F32)
            c_len = [np.zeros(C, np.int64) for _ in conds]
            c_n = [np.zeros(C, np.int64) for _ in conds]
            c_mx = [np.zeros(C, np.int64) for _ in conds]
            r_acc = [np.zeros(C, np.int64) for _ in runs]
            m_rs, m_best = np.zeros(C), np.zeros(C)
            q = [np.zeros(C) for _ in sums]
            for t in range(poff[p], poff[p + 1]):
                v = x[t]
                ok = v == v
                nok += ok
                s = s + np.where(ok, v.astype(np.float64), 0.0)
                mn = np.fmin(mn, v)
                mx = np.fmax(mx, v)
                cf, fin = [], []
                for j, (sgn, thr, _) in enumerate(conds):
                    c = sgn * v > thr
                    cf.append(c)
                    fin.append(np.where(c, 0, c_len[j]))          # length of the run that ends at this step
                    c_len[j] = np.where(c, c_len[j] + 1, 0)
                    c_n[j] += c
                    c_mx[j] = np.maximum(c_mx[j], c_len[j])
                for k, (j, w, kind) in enumerate(runs):
                    L = fin[j]
                    r_acc[k] += np.where(L >= w, L if kind == 0 else 1, 0)
                if nm:
                    e = (m_sgn * (v - m_thr0)).astype(np.float64)     # float32 excess, widened
                    m_best = np.where(fin[0] >= m_w, np.fmax(m_best, m_rs), m_best)
                    m_rs = np.where(cf[0], m_rs + e, 0.0)
                for k, (mode, sgn, thr, off_sgn, off) in enumerate(sums):
                    if mode == 0:
                        d = np.fmax(off_sgn * (v - off), F32(0))
                        q[k] = q[k] + np.where(ok, d.astype(np.float64), 0.0)
                    else:
                        q[k] = q[k] + np.where(sgn * v > thr, v.astype(np.float64), 0.0)
            res["sum"][p] = s
            res["mean"][p] = np.where(nok > 0, s / np.maximum(nok, 1), np.nan)
            res["min"][p] = np.where(nok > 0, mn, np.nan)
            res["max"][p] = np.where(nok > 0, mx, np.nan)
            for j, (_, _, wmax) in enumerate(conds):
                res[("n", j)][p] = c_n[j]
                res[("max", j)][p] = np.where(c_mx[j] >= wmax, c_mx[j], 0)
            for k, (j, w, kind) in enumerate(runs):     # the run closed by the period end
                L = c_len[j]
                res[("run", k)][p] = r_acc[k] + np.where(L >= w, L if kind == 0 else 1, 0)
            if nm:
                res[("msum", 0)][p] = np.where(c_len[0] >= m_w, np.fmax(m_best, m_rs), m_best)
            for k in range(ns):
                res[("qsum", k)][p] = q[k]
    return res


def output_slots(plan):
    """{output key of ``period_multi_raw``: slot} for the outputs the plan writes (slot >= 0)."""
    out = {"sum": plan.slot_sum, "mean": plan.slot_mean, "min": plan.slot_min, "max": plan.slot_max}
    for j in range(plan.n_cond):
        out[("n", j)] = plan.cond[j].slot_n
        out[("max", j)] = plan.cond[j].slot_max
    for k in range(plan.n_runs):
        out[("run", k)] = plan.runs[k].slot
    for k in range(plan.n_msum):
        out[("msum", k)] = plan.msum[k].slot
    for k in range(plan.n_sums):
        out[("qsum", k)] = plan.sums[k].slot
    return {k: int(s) for k, s in out.items() if s >= 0}


def is_count(key):
    return isinstance(key, tuple) and key[0] == "n"


def period_multi(x, poff, plan, n_slots):
    """The ``(max(1, n_slots), P, C)`` float32 slot buffer of ``xc_period_multi_f32`` (count slots hold int32 bits);
    slots the plan does not write are 0.  A slot named by several outputs holds the last one the kernel stores
    (sum, mean, min, max, then per condition n and max, run outputs, the run sum, conditional sums)."""
    raw = period_multi_raw(x, poff, plan)
    P, C = len(poff) - 1, np.asarray(x).shape[1]
    out = np.zeros((max(1, n_slots), P, C), F32)
    with np.errstate(over="ignore"):           # float64 sums beyond float32 round to +-inf, as in the kernel
        for key, slot in output_slots(plan).items():
            v = raw[key]
            out[slot] = v.astype(np.int32).view(F32) if is_count(key) else v.astype(F32)
    return out
