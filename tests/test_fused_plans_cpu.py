"""CPU checks of the fused multi-output pass around its kernel: the plan packer of ``indices.run_batch``
(``_PassBuilder``), the condition normalisation, the launch plan of the entry point and the sequential
oracle of oracle/multi_oracle.py against the reference-semantics compositions of oracle/xclim_oracle.py."""
import numpy as np
import pytest

import fake_device
from dispatch_host_build import multi_errors as plan_errors, multi_shape as multi_kernel
from oracle import multi_oracle as MO
from oracle import xclim_oracle as O
from xb_helpers import empty_plan, instantiations, make_field
from xclim_b200 import _lib, device
from xclim_b200.indices import _PassBuilder

F32 = np.float32
OPS = (">", "<", ">=", "<=")
FMAX = float(np.finfo(F32).max)


def _poff(rng, T, lo=1, hi=40):
    cuts = [0]
    while cuts[-1] < T:
        cuts.append(min(T, cuts[-1] + int(rng.integers(lo, hi + 1))))
    return np.asarray(cuts, np.int32)


def _data(rng, T, C, nan=0.05):
    """A persistent walk on a 0.1 grid (long runs, values on the thresholds) with NaN."""
    x = np.clip(np.cumsum(rng.choice([-0.1, 0.0, 0.1], size=(T, C), p=[0.3, 0.4, 0.3]), axis=0), -2.5, 2.5)
    x = np.round(x, 1).astype(F32)
    x[rng.random(x.shape) < nan] = np.nan
    x[:, 0] = np.nan if C > 1 else x[:, 0]
    return x


# ---------------------------------------------------------------------------------------------- dispatch
def _plan(n_cond=0, n_runs=0, n_msum=0, n_sums=0):
    p = empty_plan()
    p.n_cond, p.n_runs, p.n_msum, p.n_sums = n_cond, n_runs, n_msum, n_sums
    return p


@pytest.mark.parametrize("counts,kernel", [
    ((0, 0, 0, 0), (0, 0, 0, 0, 4, 8)),
    ((1, 0, 0, 0), (2, 0, 0, 0, 4, 8)),
    ((2, 0, 0, 0), (2, 0, 0, 0, 4, 8)),
    ((0, 0, 0, 1), (0, 0, 0, 3, 2, 12)),
    ((3, 0, 0, 0), (4, 0, 0, 0, 2, 12)),
    ((1, 0, 1, 0), (2, 0, 1, 0, 2, 12)),
    ((2, 2, 0, 0), (2, 1, 0, 0, 2, 12)),
    ((2, 4, 0, 0), (2, 2, 0, 0, 2, 12)),
    ((5, 4, 1, 2), (6, 2, 1, 3, 2, 12)),
    ((6, 2, 0, 3), (6, 1, 0, 3, 2, 12)),
])
def test_multi_dispatch_pinned(counts, kernel):
    assert multi_kernel(_plan(*counts)) == kernel


def test_multi_instantiation_list():
    inst = instantiations()
    assert len(inst) == len(set(inst)) == 38
    shapes = {(nc, ncr, nm, ns): multi_kernel(_plan(nc, 2 * ncr, nm, min(ns, 1)))[4:] for nc, ncr, nm, ns in inst}
    assert sorted(k for k, v in shapes.items() if v == (4, 8)) == [(0, 0, 0, 0), (2, 0, 0, 0)]


# ------------------------------------------------------------------------------ condition normalisation
def _float32_classes():
    tiny = np.finfo(F32).smallest_subnormal
    base = [0.0, -0.0, float(tiny), -float(tiny), 1e-40, -1e-40, 1.0, -1.0, 0.1, FMAX, -FMAX, np.inf, -np.inf]
    vals = set()
    for b in base:
        f = F32(b)
        with np.errstate(over="ignore"):
            vals.update([f, np.nextafter(f, F32(np.inf)), np.nextafter(f, F32(-np.inf))])
    return np.array(sorted(vals, key=lambda v: (float(v), np.signbit(v))) + [np.nan], F32)


@pytest.mark.parametrize("op", OPS)
def test_normalise_condition_every_float32_class(op):
    """x op t  <=>  sgn * x > thr' for every float32 class of x and t (Python floats that round to +-inf in
    float32 included); the two conditions no strict > expresses raise."""
    x = _float32_classes()
    thresholds = [float(v) for v in x] + [1e300, -1e300, 1e-50, -1e-50]
    for t in thresholds:
        with np.errstate(over="ignore"):
            t32 = F32(t)
        if (op == ">=" and t32 == -np.inf) or (op == "<=" and t32 == np.inf):
            with pytest.raises(NotImplementedError):
                device.normalise_condition(_lib.OPS[op], t)
            with pytest.raises(NotImplementedError):
                _PassBuilder().cond(_lib.OPS[op], t)
            continue
        sgn, thr = device.normalise_condition(_lib.OPS[op], t)
        with np.errstate(invalid="ignore", over="ignore"):
            got = F32(sgn) * x > F32(thr)
            exp = O.compare(x, op, t32)
        np.testing.assert_array_equal(got, exp, err_msg=f"x {op} {t!r}")


def test_run_batch_leaves_unexpressible_conditions_to_the_single_calls(monkeypatch):
    """A condition the fused pass cannot express sends its indicator to the one-call-per-indicator path."""
    from xclim_b200 import indices
    fake_device.install(monkeypatch)
    rng = np.random.default_rng(5)
    tas = (270 + 10 * rng.standard_normal((365 * 2, 2, 3))).astype(F32)
    fields = {"tasmin": make_field(tas, "2001-01-01", calendar="noleap", units="K"),
              "tasmax": make_field(tas + 5, "2001-01-01", calendar="noleap", units="K")}
    names = ["frost_days", "tn_min", "maximum_consecutive_frost_days", "ice_days", "tx_max"]
    ref = indices.run_batch(fields, names=names)

    def refuse(op_code, thr):
        raise NotImplementedError("refused")
    monkeypatch.setattr(device, "normalise_condition", refuse)
    launches = []
    real = device.period_multi
    monkeypatch.setattr(device, "period_multi", lambda *a: launches.append(a[2]) or real(*a))
    got = indices.run_batch(fields, names=names)
    for nm in names:
        np.testing.assert_array_equal(got[nm].values, ref[nm].values, err_msg=nm)
        assert got[nm].attrs == ref[nm].attrs
    # only the plain statistics are left in the fused passes: one launch per variable, no conditions
    assert len(launches) == 2 and all(p.n_cond == 0 for p in launches)


# ------------------------------------------------------------------------------------------ the packer
def _random_requests(rng):
    """A _PassBuilder with seeded random requests and {request key: expected output function}."""
    pb = _PassBuilder()
    origin = {}                                   # condition key -> (op, t)
    n_cond = int(rng.integers(1, 11))
    while len(origin) < n_cond:
        op, t = OPS[int(rng.integers(4))], float(np.round(rng.uniform(-2, 2), 1))
        c, key = pb.cond(_lib.OPS[op], t)
        origin.setdefault(key, (op, t))
        c["n"], c["max"] = bool(rng.random() < 0.5), bool(rng.random() < 0.5)
    keys = list(origin)
    for key in rng.permutation(len(keys))[:int(rng.integers(0, 5))]:
        c = pb.conds[keys[key]]
        for _ in range(int(rng.integers(1, 6))):
            c["runs"].add((("sum", "count")[int(rng.integers(2))], int(rng.integers(1, 7))))
    if rng.random() < 0.7:                       # a largest-run-sum owner (a > condition), with or without runs
        gts = [k for k in keys if origin[k][0] == ">"]
        if gts and rng.random() < 0.6:
            key = gts[int(rng.integers(len(gts)))]
        else:
            t = float(np.round(rng.uniform(-2, 2), 1)) + 0.05
            c, key = pb.cond(_lib.OPS[">"], t)
            origin.setdefault(key, (">", t))
        pb.conds[key]["ms"] = (int(rng.integers(1, 5)), 1.0, float(F32(origin[key][1])))
    for _ in range(int(rng.integers(0, 8))):
        if rng.random() < 0.5:
            pb.sums[(0, 0.0, 0.0, float(rng.choice([-1.0, 1.0])), float(F32(np.round(rng.uniform(-2, 2), 1))))] = True
        else:
            key = keys[int(rng.integers(len(keys)))]
            pb.sums[(1, key[0], key[1], 0.0, 0.0)] = True
    for st in ("sum", "mean", "min", "max"):
        if rng.random() < 0.5:
            pb.stats[st] = True
    return pb, origin


def _requested(pb):
    req = {("stat", st) for st in pb.stats}
    for key, c in pb.conds.items():
        if c["n"]:
            req.add(("n",) + key)
        if c["max"]:
            req.add(("max",) + key)
        req.update((kind,) + key + (w,) for kind, w in c["runs"])
        if c["ms"] is not None:
            req.add(("ms",) + key + (c["ms"][0],))
    req.update(("qsum",) + k for k in pb.sums)
    return req


def _expected(req, x, poff, origin):
    """The output a request asks for, from the reference-semantics compositions of the oracle."""
    x64 = x.astype(np.float64)
    with np.errstate(invalid="ignore"):
        if req[0] == "stat":
            return O.resample_reduce(x64, poff, req[1])
        if req[0] == "qsum":
            mode, sgn, thr, off_sgn, off = req[1:]
            if mode == 0:
                d = np.clip((x - F32(off)) if off_sgn > 0 else (F32(off) - x), 0, None)
                return O.resample_reduce(d.astype(np.float64), poff, "sum")
            op, t = origin[(sgn, thr)]
            return O.resample_reduce(np.where(O.compare(x, op, t), x64, np.nan), poff, "sum")
        op, t = origin[req[1:3]]
        cond = O.compare(x, op, t)
        if req[0] == "n":
            return O.threshold_count(x, op, t, poff)
        if req[0] == "max":
            return O.resample_and_rl(cond, True, O.rle_statistics, poff=poff, reducer="max", window=1)
        if req[0] in ("sum", "count"):
            return O.resample_and_rl(cond, True, O.rle_statistics, poff=poff, reducer=req[0], window=req[3])
        assert req[0] == "ms" and op == ">"
        exc = np.where(cond, x - F32(t), F32(0)).astype(np.float64)
        return O.resample_and_rl(exc, True, O.windowed_max_run_sum, req[3], poff=poff)


@pytest.mark.parametrize("seed", range(40))
def test_packer_random_requests(seed):
    rng = np.random.default_rng(1000 + seed)
    pb, origin = _random_requests(rng)
    req = _requested(pb)
    T, C = 160, 6
    x = _data(rng, T, C)
    poff = _poff(rng, T)
    seen = {}
    for i, (plan, n, where) in enumerate(pb.plans()):
        assert plan_errors(plan, n) == [], (seed, i)
        assert multi_kernel(plan)[:4] in instantiations()
        assert sorted(s for s, _ in where.values()) == list(range(n))       # one slot per request, none idle
        assert set(MO.output_slots(plan).values()) == set(range(n))
        buf = MO.period_multi(x, poff, plan, n)
        for key, (slot, is_int) in where.items():
            assert key not in seen, key                                    # each request in exactly one plan
            seen[key] = buf[slot].view(np.int32) if is_int else buf[slot]
            assert is_int == (key[0] == "n")
    assert set(seen) == req
    for key, got in seen.items():
        exp = _expected(key, x, poff, origin)
        if key[0] in ("stat", "qsum", "ms") and key[:2] not in (("stat", "min"), ("stat", "max")):
            np.testing.assert_allclose(got, exp.astype(F32), rtol=1e-6, atol=1e-9, equal_nan=True, err_msg=str(key))
        else:
            np.testing.assert_array_equal(got, np.asarray(exp).astype(got.dtype), err_msg=str(key))


def test_packer_max_sum_owner_without_runs_and_two_run_owners():
    """A largest-run-sum owner without runs takes run place 0: with two other run owners the pass needs two
    plans (one plan with three run places wrote past the end of the run outputs)."""
    pb = _PassBuilder()
    c, k25 = pb.cond(_lib.OPS[">"], 25.0)
    c["ms"] = (3, 1.0, 25.0)
    c, k30 = pb.cond(_lib.OPS[">"], 30.0)
    c["runs"].add(("sum", 6))
    c, k0 = pb.cond(_lib.OPS["<"], 0.0)
    c["runs"].add(("count", 5))
    plans = pb.plans()
    assert len(plans) == 2
    for plan, n, _ in plans:
        assert plan_errors(plan, n) == []
    first = plans[0][0]
    assert (first.cond[0].sgn, first.cond[0].thr) == k25 and first.n_msum == 1 and first.n_runs == 4
    assert first.runs[0].slot == first.runs[1].slot == -1
    assert set(plans[0][2]) | set(plans[1][2]) == _requested(pb)


# ------------------------------------------------------------- the sequential oracle, cross-checked
def _hand_plan(rng, n_cond, n_runs, n_msum, n_sums):
    """A plan over conditions drawn as (op, t) pairs: -> (plan, {condition index: (op, t)}, ms (op, t))."""
    plan = _plan(n_cond, n_runs, n_msum, n_sums)
    origin, slot = {}, 0
    for j in range(n_cond):
        op, t = OPS[int(rng.integers(4))], float(np.round(rng.uniform(-2, 2), 1))
        if j == 0 and n_msum:
            op = (">", "<")[int(rng.integers(2))]
        origin[j] = (op, t)
        e = plan.cond[j]
        e.sgn, e.thr = device.normalise_condition(_lib.OPS[op], t)
        e.wmax, e.slot_n, e.slot_max = int(rng.integers(1, 5)), slot, slot + 1
        slot += 2
    for k in range(n_runs):
        r = plan.runs[k]
        r.cond, r.window, r.kind, r.slot = k // 2, int(rng.integers(1, 8)), int(rng.integers(2)), slot
        slot += 1
    if n_msum:
        op, t = origin[0]
        m = plan.msum[0]
        m.cond, m.window, m.sgn, m.thr0, m.slot = 0, int(rng.integers(1, 5)), 1.0 if op == ">" else -1.0, t, slot
        slot += 1
    for k in range(n_sums):
        e = plan.sums[k]
        op, t = OPS[int(rng.integers(4))], float(np.round(rng.uniform(-2, 2), 1))
        e.mode, e.slot = int(rng.integers(2)), slot
        e.sgn, e.thr = device.normalise_condition(_lib.OPS[op], t)
        e.off_sgn, e.off = float(rng.choice([-1.0, 1.0])), float(F32(t))
        origin[("sum", k)] = (op, t)
        slot += 1
    plan.slot_sum, plan.slot_mean, plan.slot_min, plan.slot_max = slot, slot + 1, slot + 2, slot + 3
    return plan, origin, slot + 4


@pytest.mark.parametrize("seed", range(12))
def test_multi_oracle_matches_reference_compositions(seed):
    """oracle/multi_oracle.py (sequential, the kernel's arithmetic) against the reference-semantics
    compositions: 1e-12 relative for the float64 sums, exact for everything else."""
    rng = np.random.default_rng(seed)
    T, C = 300, 7
    x = _data(rng, T, C)
    x[40:80, 3] = 1.5                              # one run covering whole periods
    poff = _poff(rng, T, 1, 60)
    counts = (int(rng.integers(1, 7)), 2 * int(rng.integers(0, 3)), int(rng.integers(0, 2)), int(rng.integers(0, 4)))
    counts = (counts[0], min(counts[1], 2 * counts[0]), counts[2], counts[3])
    plan, origin, n = _hand_plan(rng, *counts)
    raw = MO.period_multi_raw(x, poff, plan)
    x64 = x.astype(np.float64)
    rel = dict(rtol=1e-12, atol=0, equal_nan=True)
    np.testing.assert_allclose(raw["sum"], O.resample_reduce(x64, poff, "sum"), **rel)
    np.testing.assert_allclose(raw["mean"], O.resample_reduce(x64, poff, "mean"), **rel)
    np.testing.assert_array_equal(raw["min"], O.resample_reduce(x64, poff, "min"))
    np.testing.assert_array_equal(raw["max"], O.resample_reduce(x64, poff, "max"))
    conds = []
    for j in range(plan.n_cond):
        op, t = origin[j]
        cond = O.compare(x, op, t)
        conds.append(cond)
        np.testing.assert_array_equal(raw[("n", j)], O.threshold_count(x, op, t, poff))
        m = O.resample_and_rl(cond, True, O.rle_statistics, poff=poff, reducer="max", window=1)
        np.testing.assert_array_equal(raw[("max", j)], np.where(m >= plan.cond[j].wmax, m, 0))
    for k in range(plan.n_runs):
        r = plan.runs[k]
        exp = O.resample_and_rl(conds[k // 2], True, O.rle_statistics, poff=poff,
                                reducer=("sum", "count")[r.kind], window=r.window)
        np.testing.assert_array_equal(raw[("run", k)], exp)
    if plan.n_msum:
        op, t = origin[0]
        exc = np.where(conds[0], (x - F32(t)) if op == ">" else (F32(t) - x), F32(0)).astype(np.float64)
        exp = O.resample_and_rl(exc, True, O.windowed_max_run_sum, plan.msum[0].window, poff=poff)
        np.testing.assert_allclose(raw[("msum", 0)], exp, **rel)
    for k in range(plan.n_sums):
        e = plan.sums[k]
        op, t = origin[("sum", k)]
        with np.errstate(invalid="ignore"):
            if e.mode == 0:
                d = np.clip((x - F32(e.off)) if e.off_sgn > 0 else (F32(e.off) - x), 0, None).astype(np.float64)
            else:
                d = np.where(O.compare(x, op, t), x64, np.nan)
        np.testing.assert_allclose(raw[("qsum", k)], O.resample_reduce(d, poff, "sum"), **rel)
    # the slot buffer: float32 roundings of the above, counts as int32 bits
    buf = MO.period_multi(x, poff, plan, n)
    np.testing.assert_array_equal(buf[plan.cond[0].slot_n].view(np.int32) if plan.n_cond else 0,
                                  raw[("n", 0)].astype(np.int32) if plan.n_cond else 0)
    np.testing.assert_array_equal(buf[plan.slot_mean], raw["mean"].astype(F32))


def test_multi_oracle_empty_and_all_nan_periods():
    x = np.full((6, 4), np.nan, F32)
    x[3:, 1] = 2.0
    poff = np.array([0, 0, 3, 3, 6], np.int32)      # periods 0 and 2 are empty
    plan, _, _ = _hand_plan(np.random.default_rng(0), 2, 2, 1, 2)
    raw = MO.period_multi_raw(x, poff, plan)
    assert (raw["sum"][[0, 1, 2]] == 0).all() and (raw[("n", 0)][[0, 1, 2]] == 0).all()
    assert np.isnan(raw["mean"][[0, 1, 2]]).all() and np.isnan(raw["min"][:, 0]).all()
    assert raw["max"][3, 1] == 2.0 and raw["mean"][3, 1] == 2.0
    for k in range(plan.n_sums):
        assert (raw[("qsum", k)][[0, 1, 2]] == 0).all()
