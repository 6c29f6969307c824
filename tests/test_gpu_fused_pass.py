"""The fused multi-output pass (`xc_period_multi_f32`, csrc/period_stats.cu) on hand-built plans, bit for bit
against the sequential restatement of oracle/multi_oracle.py: every `period_multi_kernel<NC, NCR, NM, NS, VEC,
UNROLL>` instantiation (named through the launch plan the entry point executes), hostile data, grid edges and
the plan checks; then `indices.run_batch` on the plan shapes and grids the default batch never builds."""
import ctypes

import numpy as np
import pytest

from dispatch_host_build import multi_errors as plan_errors, multi_shape as multi_kernel
from oracle import multi_oracle as MO
from xb_helpers import empty_plan, instantiations
from xclim_b200 import _lib, device

pytestmark = pytest.mark.gpu


F32 = np.float32
FMAX = float(np.finfo(F32).max)
TINY = float(np.finfo(F32).smallest_subnormal)
OPS = (">", "<", ">=", "<=")
# thresholds on the data grid, at signed zeros, subnormals, the float32 extremes and the infinities
THRESHOLDS = [0.0, -0.0, 0.5, -1.0, 1.5, 2.0, TINY, -1e-40, FMAX, -FMAX, np.inf, -np.inf]


def _neighbours(vals):
    out = []
    with np.errstate(over="ignore"):
        for v in vals:
            f = F32(v)
            out += [f, np.nextafter(f, F32(np.inf)), np.nextafter(f, F32(-np.inf))]
    return out


SPECIALS = np.array(_neighbours(THRESHOLDS) + [np.nan, np.inf, -np.inf, 0.0, -0.0, TINY, -TINY, 1e-40, FMAX, -FMAX,
                                               3.4e38, -3.4e38], F32)


def _poff(rng, T):
    """Period offsets with lengths 0 to 13 (the remainder loops after 8 and 12 rows in flight), and longer."""
    lens = []
    while sum(lens) < T:
        lens.append(int(rng.choice([0, 1, 2, 3, 5, 7, 8, 9, 11, 12, 13, 24, 25, 40])))
    poff = np.concatenate([[0], np.minimum(np.cumsum(lens), T)]).astype(np.int32)
    poff[-1] = T
    return poff


def _hostile(rng, T, C, poff):
    """A persistent walk on a 0.5 grid (runs across period edges, values on the thresholds) with the special
    values sprinkled in, a constant cell (runs covering whole periods), an all-NaN cell and all-NaN periods."""
    x = np.cumsum(rng.choice([-0.5, 0.0, 0.5], size=(T, C), p=[0.25, 0.5, 0.25]), axis=0)
    x = np.clip(x, -2.5, 2.5).astype(F32)
    hit = rng.random((T, C)) < 0.12
    x[hit] = rng.choice(SPECIALS, size=int(hit.sum()))
    if C >= 8:
        x[:, 0] = 1.5
        x[:, 1] = np.nan
        x[:, -1] = 2.0             # runs over whole periods and across period edges, and (every other period
        starts = poff[:-1][::2]    # starting below the thresholds) runs that end on the period's last step
        x[starts[starts < T], -1] = -2.0
    for p in rng.choice(len(poff) - 1, size=min(3, len(poff) - 1), replace=False):
        x[poff[p]:poff[p + 1], rng.integers(C)] = np.nan
    return x


def _cond(rng):
    while True:
        op, t = OPS[int(rng.integers(4))], THRESHOLDS[int(rng.integers(len(THRESHOLDS)))]
        if not ((op == ">=" and t == -np.inf) or (op == "<=" and t == np.inf)):
            return device.normalise_condition(_lib.OPS[op], t), t


def random_plan(rng, nc, ncr, nm, ns, n_cond=None):
    """A plan of the (NC, NCR, NM, NS) instantiation with actual counts below the rounded ones where possible
    (computed-and-dropped entries), slots in a random order, some shared, some left at -1."""
    if n_cond is None:
        lo = {0: 0, 2: 1, 4: 3, 6: 5}[nc]
        n_cond = int(rng.integers(max(lo, ncr, nm), nc + 1))
    plan = empty_plan()
    plan.n_cond, plan.n_runs, plan.n_msum = n_cond, 2 * ncr, nm
    plan.n_sums = int(rng.integers(1, 4)) if ns else 0
    outs = []                                        # setters of every output slot
    for j in range(n_cond):
        e = plan.cond[j]
        (e.sgn, e.thr), _ = _cond(rng)
        e.wmax = int(rng.choice([1, 1, 2, 3, 5]))
        outs += [lambda s, e=e: setattr(e, "slot_n", s), lambda s, e=e: setattr(e, "slot_max", s)]
    for k in range(2 * ncr):
        r = plan.runs[k]
        r.cond, r.window, r.kind = k // 2, int(rng.choice([1, 2, 3, 4, 7, 20, 100000])), int(rng.integers(2))
        outs.append(lambda s, r=r: setattr(r, "slot", s))
    if nm:
        m = plan.msum[0]
        m.cond, m.window = 0, int(rng.choice([1, 2, 3, 6]))
        if rng.random() < 0.5:                       # the hot_spell_max_magnitude shape: excess over condition 0
            m.sgn, m.thr0 = plan.cond[0].sgn, plan.cond[0].sgn * plan.cond[0].thr
        else:
            m.sgn, m.thr0 = float(rng.choice([-1.0, 1.0])), float(F32(THRESHOLDS[int(rng.integers(len(THRESHOLDS)))]))
        outs.append(lambda s, m=m: setattr(m, "slot", s))
    for k in range(plan.n_sums):
        e = plan.sums[k]
        e.mode = int(rng.integers(2))
        (e.sgn, e.thr), t = _cond(rng)
        e.off_sgn, e.off = float(rng.choice([-1.0, 1.0])), float(F32(t)) if rng.random() < 0.7 else 0.25
        outs.append(lambda s, e=e: setattr(e, "slot", s))
    for name in ("slot_sum", "slot_mean", "slot_min", "slot_max"):
        outs.append(lambda s, name=name: setattr(plan, name, s))
    order = rng.permutation(len(outs))
    n = 0
    for i in order:
        u = rng.random()
        if u < 0.15:
            outs[i](-1)
        elif u < 0.25 and n:
            outs[i](int(rng.integers(n)))            # shares a slot: the kernel's last store wins
        else:
            outs[i](n)
            n += 1
    return plan, n


def _assert_matches_oracle(buf, x, poff, plan, what=""):
    """Every slot the plan writes, bit for bit (any NaN matches any NaN; min / max: +0 == -0)."""
    raw = MO.period_multi_raw(x, poff, plan)
    last = {}
    for key, slot in MO.output_slots(plan).items():
        last[slot] = key
    assert last, "plan writes nothing"
    for slot, key in last.items():
        got = buf[slot]
        if MO.is_count(key):
            np.testing.assert_array_equal(got.view(np.int32), raw[key].astype(np.int32), err_msg=f"{what} {key}")
            continue
        with np.errstate(over="ignore"):
            exp = raw[key].astype(F32)
        nan = np.isnan(exp)
        np.testing.assert_array_equal(np.isnan(got), nan, err_msg=f"{what} {key}: NaN positions")
        if key in ("min", "max"):
            np.testing.assert_array_equal(got[~nan], exp[~nan], err_msg=f"{what} {key}")
        else:
            bad = got.view(np.uint32)[~nan] != exp.view(np.uint32)[~nan]
            assert not bad.any(), f"{what} {key}: {int(bad.sum())} values differ, e.g. " \
                                  f"{got[~nan][bad][:4]} vs {exp[~nan][bad][:4]}"


def _run(x_dev, poff, plan, n):
    import torch
    buf = device.period_multi(x_dev, poff, plan, n)
    torch.cuda.synchronize()
    return buf.cpu().numpy()


# ------------------------------------------------------------------------------------ every instantiation
@pytest.mark.parametrize("inst", instantiations(), ids=lambda i: "NC%d_NCR%d_NM%d_NS%d" % i)
def test_every_instantiation_hostile_data(inst, cuda):
    import torch
    nc, ncr, nm, ns = inst
    rng = np.random.default_rng(hash(inst) % 2**32)
    T = 400
    C = int(rng.choice([4, 8, 12, 256, 260]))
    poff = _poff(rng, T)
    x = _hostile(rng, T, C, poff)
    for rep in range(2):                             # two plans per instantiation
        plan, n = random_plan(rng, *inst)
        assert plan_errors(plan, n) == []
        k = multi_kernel(plan)
        assert k[:4] == inst
        assert k[4:] == ((4, 8) if (ncr, nm, ns) == (0, 0, 0) and nc <= 2 else (2, 12))
        buf = _run(torch.from_numpy(x).to(cuda), poff, plan, n)
        _assert_matches_oracle(buf, x, poff, plan, f"<{nc},{ncr},{nm},{ns},{k[4]},{k[5]}> C={C} plan {rep}")


@pytest.mark.parametrize("inst", [(2, 0, 0, 0), (6, 2, 1, 3)], ids=["vec4_unroll8", "vec2_unroll12"])
def test_long_series_many_periods(inst, cuda):
    """T of a few thousand steps in a few hundred periods, windows longer than the period included."""
    import torch
    rng = np.random.default_rng(77 + inst[0])
    T, C = 3000, 68
    poff = _poff(rng, T)
    assert len(poff) - 1 >= 200
    x = _hostile(rng, T, C, poff)
    plan, n = random_plan(rng, *inst, n_cond=inst[0])
    assert multi_kernel(plan)[:4] == inst
    _assert_matches_oracle(_run(torch.from_numpy(x).to(cuda), poff, plan, n), x, poff, plan)


# ------------------------------------------------------------------------------------------ grid edges
@pytest.mark.parametrize("C", [4, 8, 252, 256, 260, 508, 512, 516, 4100])
@pytest.mark.parametrize("inst", [(2, 0, 0, 0), (4, 2, 1, 3)], ids=["vec4_unroll8", "vec2_unroll12"])
def test_grid_edges(C, inst, cuda):
    """C just below, at and above one CTA of either launch shape (512 cells with 4 per thread, 256 with 2), and
    a few thousand cells with a partial last CTA; the last cells are always compared."""
    import torch
    rng = np.random.default_rng(C * 7 + inst[0])
    T = 90
    poff = _poff(rng, T)
    x = _hostile(rng, T, C, poff)
    plan, n = random_plan(rng, *inst)
    _assert_matches_oracle(_run(torch.from_numpy(x).to(cuda), poff, plan, n), x, poff, plan, f"C={C}")


@pytest.mark.parametrize("inst", [(2, 0, 0, 0), (6, 1, 1, 3)], ids=["vec4_unroll8", "vec2_unroll12"])
@pytest.mark.parametrize("C,off,width", [(8, 4, 20), (256, 8, 300), (516, 12, 540)])
def test_strided_views(C, off, width, inst, cuda):
    """ldx > C: a column block at a 16-byte aligned offset inside a wider buffer, read in place."""
    import torch
    rng = np.random.default_rng(C + off)
    T = 120
    poff = _poff(rng, T)
    wide = _hostile(rng, T, width, poff)
    x_dev = torch.from_numpy(wide).to(cuda)[:, off:off + C]
    assert x_dev.stride(0) == width and x_dev.data_ptr() % 16 == 0
    plan, n = random_plan(rng, *inst)
    _assert_matches_oracle(_run(x_dev, poff, plan, n), wide[:, off:off + C], poff, plan, f"ldx={width}")


@pytest.mark.parametrize("C,ldx,off", [(5, 5, 0), (3, 3, 0), (1, 1, 0), (35, 35, 0), (8, 10, 0), (8, 12, 1)])
def test_unaligned_grids_are_padded(C, ldx, off, cuda):
    """device.period_multi runs grids the kernel cannot read four cells at a time (C or ldx not a multiple of 4, a
    start 4 bytes past 16-byte alignment) on a zero-padded copy: the same results."""
    import torch
    rng = np.random.default_rng(C + ldx + off)
    T = 70
    poff = _poff(rng, T)
    flat = torch.from_numpy(_hostile(rng, T * ldx + 4, 1, poff).reshape(-1)).to(cuda)
    x_dev = flat[off:off + T * ldx].reshape(T, ldx)[:, :C]
    assert (x_dev.data_ptr() % 16 != 0) == (off != 0)
    x_h = x_dev.cpu().numpy()
    for inst in [(2, 0, 0, 0), (6, 2, 1, 3)]:
        plan, n = random_plan(rng, *inst)
        buf = _run(x_dev, poff, plan, n)
        assert buf.shape == (max(1, n), len(poff) - 1, C)
        _assert_matches_oracle(buf, x_h, poff, plan, f"C={C} ldx={x_dev.stride(0)}")


# ------------------------------------------------------------------------------------------ ABI rejections
def _call(x, T, C, ldx, poff_d, P, plan, out, n_slots):
    import torch
    torch.cuda.synchronize()
    return _lib.load().xc_period_multi_f32(x, T, C, ldx, poff_d.data_ptr(), P, ctypes.byref(plan), out.data_ptr(),
                                           n_slots, 0)


def _ok_plan():
    plan = empty_plan()
    plan.n_cond, plan.n_runs, plan.n_msum, plan.n_sums = 2, 2, 1, 1
    plan.cond[0].sgn, plan.cond[0].thr, plan.cond[0].slot_n = 1.0, 0.5, 0
    plan.cond[1].sgn, plan.cond[1].thr = -1.0, 0.0
    plan.runs[0].window, plan.runs[0].slot = 2, 1
    plan.msum[0].window, plan.msum[0].sgn, plan.msum[0].slot = 1, 1.0, 2
    plan.sums[0].slot = 3
    plan.slot_mean = 4
    return plan


def _bad(mutate):
    plan = _ok_plan()
    mutate(plan)
    return plan


BAD_PLANS = {
    "odd_n_runs": (lambda p: setattr(p, "n_runs", 1), "an even number"),
    "run_not_at_its_place": (lambda p: setattr(p.runs[1], "cond", 1), "run output not at its condition's place"),
    "msum_cond_not_0": (lambda p: setattr(p.msum[0], "cond", 1), "run output not at its condition's place"),
    "too_many_conditions": (lambda p: setattr(p, "n_cond", 7), "at most 6 conditions"),
    "too_many_runs": (lambda p: setattr(p, "n_runs", 6), "at most 6 conditions"),
    "too_many_msums": (lambda p: setattr(p, "n_msum", 2), "at most 6 conditions"),
    "too_many_sums": (lambda p: setattr(p, "n_sums", 4), "at most 6 conditions"),
    "runs_without_conditions": (lambda p: (setattr(p, "n_cond", 0), setattr(p, "n_msum", 0)),
                                "run outputs need their condition"),
    "slot_past_n_slots": (lambda p: setattr(p, "slot_sum", 5), "output slot outside [-1, n_slots)"),
    "slot_below_minus_1": (lambda p: setattr(p.cond[1], "slot_max", -2), "output slot outside [-1, n_slots)"),
    "run_slot_past_n_slots": (lambda p: setattr(p.runs[1], "slot", 5), "output slot outside [-1, n_slots)"),
    "sum_slot_past_n_slots": (lambda p: setattr(p.sums[0], "slot", 5), "output slot outside [-1, n_slots)"),
    "window_0": (lambda p: setattr(p.runs[0], "window", 0), "window < 1"),
    "bad_sum_mode": (lambda p: setattr(p.sums[0], "mode", 2), "output slot outside"),
}


def _rejects(x_ptr, T, C, ldx, plan, n_slots, msg, cuda):
    import torch
    poff_d = torch.tensor([0, T], dtype=torch.int32, device=cuda)
    out = torch.full((max(1, n_slots), 1, max(C, 1)), 7.0, device=cuda)
    rc = _call(x_ptr, T, C, ldx, poff_d, 1, plan, out, n_slots)
    err = _lib.load().xc_last_error().decode()
    torch.cuda.synchronize()
    assert rc == _lib.XC_ERR_INVALID, (rc, err)
    assert msg in err, err
    assert (out == 7.0).all(), "a rejected call launched"


@pytest.mark.parametrize("case", sorted(BAD_PLANS))
def test_plan_rejections(case, cuda):
    import torch
    mutate, msg = BAD_PLANS[case]
    x = torch.zeros((16, 8), device=cuda)
    plan = _bad(mutate)
    assert plan_errors(plan, 5), "the plan check accepts it"
    assert plan_errors(_ok_plan(), 5) == []
    _rejects(x.data_ptr(), 16, 8, 8, plan, 5, msg, cuda)


@pytest.mark.parametrize("case", ["C_not_multiple_of_4", "ldx_not_multiple_of_4", "x_misaligned"])
def test_buffer_rejections(case, cuda):
    import torch
    x = torch.zeros((16, 16), device=cuda)
    C, ldx, ptr = {"C_not_multiple_of_4": (6, 8, x.data_ptr()), "ldx_not_multiple_of_4": (4, 6, x.data_ptr()),
                   "x_misaligned": (4, 8, x.data_ptr() + 4)}[case]
    _rejects(ptr, 16, C, ldx, _ok_plan(), 5, "needs C, ldx multiples of 4 and 16-byte aligned buffers", cuda)


def test_rejects_time_axis_of_2_pow_24(cuda):
    """Counters and run lengths are float32, exact only below 2^24 steps: a real (2^24, 4) buffer is refused."""
    import torch
    T = 1 << 24
    x = torch.zeros((T, 4), device=cuda)
    _rejects(x.data_ptr(), T, 4, 4, _ok_plan(), 5, "shorter than 2^24 steps", cuda)
    del x
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------- run_batch on the GPU
def _batch_inputs(shape, calendar, seed):
    from xb_helpers import make_field
    rng = np.random.default_rng(seed)
    start, T = ("1983-01-01", 365 * 3 + 1) if calendar == "standard" else ("1981-01-01", 365 * 3)
    t = np.arange(T)
    season = 14 * np.sin(2 * np.pi * (t % 365 - 110) / 365).reshape((T,) + (1,) * len(shape))
    tas = (278 + season + 4 * rng.standard_normal((T,) + shape)).astype(F32)
    spread = np.abs(4 + rng.standard_normal((T,) + shape)).astype(F32)
    data = {"tas": tas, "tasmax": (tas + spread).astype(F32), "tasmin": (tas - spread).astype(F32),
            "pr": rng.gamma(0.4, 6.0, size=(T,) + shape).astype(F32)}
    data["pr"][rng.random(data["pr"].shape) < 0.45] = 0
    for a in data.values():
        a[rng.random(a.shape) < 0.003] = np.nan
    units = {"tas": "K", "tasmax": "K", "tasmin": "K", "pr": "mm/d"}
    fields = {k: make_field(v, start, calendar=calendar, units=units[k]) for k, v in data.items()}
    return data, fields


def _check_batch(names, data, fields, oracle_cache):
    """run_batch(names) == the single calls bit for bit (values, dtype, dims, attrs), and the oracle at 1e-5."""
    import inspect

    from oracle import xclim_oracle as O
    from oracle.batch50 import oracle_indicator
    from xclim_b200 import calendar as xcal, indices
    per_of = {"tx90p": ("tasmax", 90.0), "tx10p": ("tasmax", 10.0), "tn90p": ("tasmin", 90.0)}
    pers = {v: xcal.select_percentile(xcal.percentile_doy(fields[v[0]], window=5, per=v[1]), v[1])
            for nm, v in per_of.items() if nm in names}
    fused = indices.run_batch(fields, pers, names=names)
    var_of = dict(indices.BATCH_INDICATORS)
    assert list(fused) == [n for n, _ in indices.BATCH_INDICATORS if n in names]
    for name in names:
        var = var_of[name]
        fn = getattr(indices, name)
        ref = fn(fields[var], pers[per_of[name]]) if name in per_of else fn(fields[var])
        got = fused[name]
        assert got.dims == ref.dims and got.values.dtype == ref.values.dtype, name
        np.testing.assert_array_equal(got.values, ref.values, err_msg=name)
        assert got.attrs == ref.attrs, name
        if name not in oracle_cache:
            da, x = fields[var], data[var]
            poff = da.time.period_offsets(inspect.signature(fn).parameters["freq"].default)
            if name in per_of:
                per = per_of[name][1]
                tab = O.percentile_doy(x, da.time.year, da.time.doy, 5, per)[:, 0]
                oracle_cache[name] = O.doy_threshold_count(x, tab, da.time.doy, poff, "<" if name == "tx10p" else ">")
            else:
                oracle_cache[name] = np.asarray(oracle_indicator(name, x, poff, da.time, data))
        exp = np.asarray(oracle_cache[name])
        assert got.values.shape == exp.shape, name
        if np.issubdtype(got.values.dtype, np.integer) or (indices.BATCH_FUSED.get(name) or ("",))[0] in ("spell", "maxlen"):
            np.testing.assert_array_equal(got.values, exp.astype(got.values.dtype), err_msg=name)
        else:
            np.testing.assert_allclose(got.values, exp, rtol=1e-5, atol=1e-6, equal_nan=True, err_msg=name)


@pytest.mark.parametrize("calendar", ["noleap", "standard"])
def test_run_batch_every_indicator_alone(calendar, cuda):
    """names=[name]: each indicator's pass alone, a plan shape of its own, on a 5 x 7 grid."""
    from xclim_b200 import indices
    data, fields = _batch_inputs((5, 7), calendar, 91)
    cache = {}
    for name, _ in indices.BATCH_INDICATORS:
        _check_batch([name], data, fields, cache)


@pytest.mark.parametrize("calendar", ["noleap", "standard"])
@pytest.mark.parametrize("shape", [(5, 7), (3, 1), (1, 1), (4, 8), (6, 10)], ids=lambda s: "%dx%d" % s)
def test_run_batch_random_subsets_and_grids(shape, calendar, cuda):
    from xclim_b200 import indices
    data, fields = _batch_inputs(shape, calendar, 17 + shape[0] * 10 + shape[1])
    all_names = [n for n, _ in indices.BATCH_INDICATORS]
    rng = np.random.default_rng(shape[0] * 100 + shape[1] + (calendar == "standard"))
    cache = {}
    _check_batch(all_names, data, fields, cache)
    for _ in range(3):
        k = int(rng.integers(2, 15))
        _check_batch([all_names[i] for i in sorted(rng.choice(len(all_names), size=k, replace=False))], data, fields,
                     cache)
