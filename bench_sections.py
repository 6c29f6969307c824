"""Sections of bench.py beyond the headline cdd kernel: full-size parity sample, NCCL gather, weak
replicas, tx90p (3a), bootstrap (3b), EQM, batch of 50, end-to-end host-buffer legs.

Every section works on THIS RANK's lat tile of the one global (10950, 721, 1440) grid, times with
CUDA events on the launching stream (warm-up first, barrier + synchronize on both sides), reduces
with MAX over ranks and reports whole-grid cells/s plus a roofline entry whose algorithmic bytes are
SURVEY.md section 8(d)'s per-cell figures times the cells of the tile.  The oracle is imported here
only as the checker / CPU-baseline leg.
"""
from __future__ import annotations

import csv
import json
import os
import time
from dataclasses import dataclass, field

import numpy as np

T_FULL, X_FULL, YEAR = 10950, 1440, 365


@dataclass
class Ctx:
    args: object
    dev: object
    rank: int
    world: int
    local: int
    barrier: object
    max_over_ranks: object
    peak: dict
    root: str
    rows: int = 0
    row0: int = 0
    n_lat_global: int = 721
    extra: dict = field(default_factory=dict)


def measured_peak(root):
    try:
        p = json.load(open(os.path.join(root, "MEASURED_PEAKS.json")))
        return {"hbm_gbs": float(p["hbm_gbs"]), "source": "MEASURED_PEAKS.json hbm_gbs (measured)"}
    except Exception:
        return {"hbm_gbs": 3350.0, "source": "H100 SXM data sheet, 3.35 TB/s (not measured)"}


def ncu_traffic(root, kernel, tile):
    """dram__bytes_read.sum + dram__bytes_write.sum per launch of `kernel` on a tile of this shape, from the
    committed table of ncu --set full captures (profiles/ncu_traffic.csv, written by tools/ncu_traffic.py from
    the .ncu-rep files); None when no capture of that kernel on that shape exists."""
    path = os.path.join(root, "profiles", "ncu_traffic.csv")
    if not os.path.exists(path):
        return None
    best = None
    for row in csv.DictReader(open(path)):
        if kernel in row["kernel"] and [int(v) for v in row["grid"].split("x")] == list(tile):
            best = float(row["dram_read_bytes"]) + float(row["dram_write_bytes"])
    return best


def roofline(ctx, alg_bytes, ms, kernel, tile=None, bound="hbm"):
    ach = alg_bytes / (ms * 1e-3) / 1e9
    r = {"bound": bound, "achieved": ach, "peak": ctx.peak["hbm_gbs"], "unit": "GB/s", "frac": ach / ctx.peak["hbm_gbs"],
         "algorithmic_bytes": alg_bytes, "launch_ms": ms, "kernel": kernel,
         "traffic": ncu_traffic(ctx.root, kernel.split("<")[0], tile) if tile else None}
    return r


def timeit(ctx, fn, steps, warmup=2):
    """mean ms per call over `steps` calls, CUDA events, MAX over ranks."""
    import torch
    for _ in range(warmup):
        fn()
    ctx.barrier()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    ev[0].record()
    for i in range(steps):
        fn()
        ev[i + 1].record()
    ctx.barrier()
    (ms,) = ctx.max_over_ranks([ev[0].elapsed_time(ev[steps]) / steps])
    return ms


def sample_cells(C, n, seed):
    """n seeded random cells + the last 256 cells (the last CTAs of every kernel), sorted unique."""
    rng = np.random.default_rng(seed)
    sel = np.unique(np.concatenate([rng.integers(0, C, size=min(n, C)), np.arange(max(0, C - 256), C), [0, 1]]))
    return sel


def tile_synth(ctx, kind, seed):
    from xclim_b200 import device
    C = ctx.rows * X_FULL
    return device.synth(T_FULL, C, kind=kind, seed=seed, cell_offset=ctx.row0 * X_FULL, cells_per_lat=X_FULL,
                        n_lat_global=ctx.n_lat_global)


# ------------------------------------------------------------------------------------------------ parity (cdd)
def parity_cdd(ctx, pr, poff, out, valid):
    """>= 4096 sampled cells of the full-size output (incl. the last CTA's cells) against the oracle."""
    import torch
    from oracle import xclim_oracle as O
    C = pr.shape[1]
    sel = sample_cells(C, 4096, 11 + ctx.rank)
    idx = torch.from_numpy(sel).to(ctx.dev)
    xs = pr[:, idx].cpu().numpy()
    exp = O.maximum_consecutive_dry_days(xs, 1.0, poff)
    ok_out = bool(np.array_equal(out[:, idx].cpu().numpy(), exp))
    ok_valid = bool(np.array_equal(valid[:, idx].cpu().numpy() != YEAR, O.missing_any(xs, poff)))
    (bad,) = ctx.max_over_ranks([0.0 if (ok_out and ok_valid) else 1.0])
    assert bad == 0.0, "full-size parity sample of maximum_consecutive_dry_days differs from the oracle"
    return {"cells_checked_per_rank": int(sel.size), "includes_last_cta": True, "cdd_bit_exact": True,
            "missing_mask_exact": True}


# ------------------------------------------------------------------------------------------------ gather
def gather_section(ctx, out, P):
    """Optional reassembly of the (P, lat, lon) result on every rank: all_gather over NCCL / NVLink."""
    from xclim_b200 import multigpu
    loc = out.view(P, ctx.rows, X_FULL)
    full = multigpu.gather_lat(loc, 1, ctx.n_lat_global)
    assert tuple(full.shape) == (P, ctx.n_lat_global, X_FULL)
    ms = timeit(ctx, lambda: multigpu.gather_lat(loc, 1, ctx.n_lat_global), 5, warmup=2)
    nbytes = P * ctx.n_lat_global * X_FULL * 4
    return {"ms": ms, "bytes_gathered_per_rank": nbytes, "gbs_per_rank": nbytes / (ms * 1e-3) / 1e9,
            "api": "xclim_b200.multigpu.gather_lat (torch.distributed.all_gather, NCCL)",
            "note": "timed separately: not part of the data path"}


# ------------------------------------------------------------------------------------------------ weak replicas
def weak_section(ctx):
    """Secondary figure: every rank a full (10950, n_lat, 1440) grid (N independent replicas)."""
    import torch
    from xclim_b200 import _lib, device
    Yg = ctx.n_lat_global
    C = Yg * X_FULL
    P = T_FULL // YEAR
    poff = np.arange(P + 1, dtype=np.int32) * YEAR
    x = device.synth(T_FULL, C, kind=0, seed=2, cell_offset=ctx.rank * C, cells_per_lat=X_FULL,
                     n_lat_global=Yg * ctx.world)
    fn = lambda: device.period_runstat(x, poff, _lib.OPS["<"], 1.0, _lib.RL_REDUCERS["max"], 1, True,  # noqa: E731
                                       want_valid=True)
    ms = timeit(ctx, fn, 5, warmup=3)
    del x
    torch.cuda.empty_cache()
    return {"value": C * ctx.world / (ms * 1e-3), "unit": "grid-cells/s", "ms_per_step": ms, "scaling": "weak",
            "note": f"{ctx.world} independent replicas of the full grid (one per GPU); not the headline"}


# ------------------------------------------------------------------------------------------------ tx90p 3a / 3b
def tx90p_sections(ctx, line, want_3a=True, want_3b=True):
    import torch
    import xclim_b200
    from oracle import xclim_oracle as O
    from xclim_b200 import Field, TimeAxis, _lib, calendar as xcal, device, indices

    args = ctx.args
    T, X = T_FULL, X_FULL
    C = ctx.rows * X
    N = T // YEAR
    poff = np.arange(N + 1, dtype=np.int32) * YEAR
    doy = (np.arange(T) % YEAR + 1).astype(np.int16)
    yidx = (np.arange(T) // YEAR).astype(np.int16)
    tasmax = tile_synth(ctx, 1, 3)
    steps = max(1, min(args.steps, 5))
    cells_total = ctx.n_lat_global * X
    sel = sample_cells(C, 64, 23 + ctx.rank)
    idx = torch.from_numpy(sel).to(ctx.dev)
    xs = tasmax[:, idx].cpu().numpy()

    if want_3a:
        run_per = lambda: device.percentile_doy(tasmax, doy, yidx, YEAR, N, 5, [90.0], 1 / 3, 1 / 3)  # noqa: E731
        table = run_per()
        run_cnt = lambda: device.doy_threshold_count(tasmax, poff, doy, table[0], _lib.OPS[">"], want_valid=True)  # noqa: E731
        t_per = timeit(ctx, run_per, steps)
        t_cnt = timeit(ctx, run_cnt, steps)
        table = run_per()
        cnt, valid = run_cnt()
        tab_o = O.percentile_doy(xs, yidx.astype(np.int64), doy.astype(np.int64), 5, 90.0)[:, 0]
        table_equal = bool(np.array_equal(tab_o, table[0][:, idx].cpu().numpy(), equal_nan=True))
        cnt_o = O.doy_threshold_count(xs, tab_o, doy.astype(np.int64), poff, ">")
        counts_equal = bool(np.array_equal(cnt_o, cnt[:, idx].cpu().numpy()))
        frac = float(cnt.double().mean().item()) / YEAR
        assert 0.07 < frac < 0.13, frac
        assert table_equal and counts_equal, (table_equal, counts_equal)
        cpu = None
        if ctx.rank == 0 and ctx.world == 1 and "cpu" in args.sections:
            ncell = 4096
            xs_cpu = tasmax[:, :ncell].cpu().numpy()
            t0 = time.perf_counter()
            tab_c = O.percentile_doy(xs_cpu, yidx.astype(np.int64), doy.astype(np.int64), 5, 90.0)[:, 0]
            O.doy_threshold_count(xs_cpu, tab_c, doy.astype(np.int64), poff, ">")
            dt = time.perf_counter() - t0
            cpu = {"value": ncell / dt, "unit": "grid-cells/s", "cores": 1, "kind": "port",
                   "sample": f"(10950, {ncell}) cells, percentile_doy + count, {dt:.1f} s"}
        alg_per = T * C * 4 + YEAR * C * 8
        alg_cnt = T * C * 4 + YEAR * C * 8 + N * C * 4 * 2
        tile = [T, ctx.rows, X]
        line["tx90p"] = {
            "workload": f"3a: percentile_doy(window=5, per=90, base=30 yr) + tx90p count on tasmax ({T},{ctx.n_lat_global},{X}) "
                        f"f32, lat-tiled over {ctx.world} rank(s)",
            "value": cells_total / ((t_per + t_cnt) * 1e-3), "unit": "grid-cells/s",
            "ms_percentile_doy": t_per, "ms_count": t_cnt, "steps": steps,
            "roofline_percentile_doy": roofline(ctx, alg_per, t_per, "percentile_doy_w5t_kernel<14> (TMA)", tile),
            "roofline_count": roofline(ctx, alg_cnt, t_cnt, "doy_count_years_kernel<GT,3,VALID>", tile),
            "gpu_launches_per_step": 2, "cpu_baseline": cpu,
            "check": {"oracle_cells_per_rank": int(sel.size), "includes_last_cta": True, "table_bit_exact": table_equal,
                      "counts_exact": counts_equal, "mean_exceedance_fraction": frac},
        }
        del table, cnt, valid

    if want_3b:
        # 3b: base = first 15 years, bootstrap=True, through the public index functions on device-resident
        # Fields (results stay in HBM): percentile_doy(base) + tx90p(bootstrap=True)
        nb = 15
        ta = TimeAxis.daily("1981-01-01", T, "noleap")
        fld = Field(tasmax.view(T, ctx.rows, X), ("time", "lat", "lon"), ta, {}, {"units": "K"})
        base = fld.isel_time(slice(0, nb * YEAR))

        def run_3b():
            with xclim_b200.set_options(device_outputs=True):
                per = xcal.select_percentile(xcal.percentile_doy(base, window=5, per=90.0), 90.0)
                return indices.tx90p(fld, per, freq="YS", bootstrap=True)

        res = run_3b()
        bsteps = max(1, min(args.steps, 3))
        ms = timeit(ctx, run_3b, bsteps, warmup=1)
        # the bootstrap kernel alone (the compute-bound part)
        step_period = np.repeat(np.arange(nb), YEAR).astype(np.int32)
        ms_k = timeit(ctx, lambda: device.bootstrap_doy_count(tasmax, 0, nb, YEAR, step_period, N, 5, 90.0, 1 / 3,
                                                              1 / 3, _lib.OPS[">"]), bsteps, warmup=1)
        got = res.values.reshape(N, C)
        ncheck = 6
        sel_b = sel[:: max(1, sel.size // ncheck)][:ncheck]
        t0 = time.perf_counter()
        exp = O.bootstrap_doy_count(tasmax[:, torch.from_numpy(sel_b).to(ctx.dev)].cpu().numpy(),
                                    (np.arange(T) // YEAR + 1981).astype(np.int64), doy.astype(np.int64), poff,
                                    (1981, 1981 + nb - 1), window=5, per=90.0, op=">")
        dt = time.perf_counter() - t0
        boot_equal = bool(np.array_equal(got[:, torch.from_numpy(sel_b).to(ctx.dev)].cpu().numpy(), exp))
        assert boot_equal, "bootstrap sample differs from the oracle"
        alg = T * C * 4 + YEAR * C * 8 + N * C * 8
        line["bootstrap"] = {
            "workload": f"3b: percentile_doy(base = first {nb} yr, window=5, per=90) + tx90p(bootstrap=True) on tasmax "
                        f"({T},{ctx.n_lat_global},{X}) f32, lat-tiled over {ctx.world} rank(s); "
                        f"{nb * (nb - 1) * YEAR} resampled quantiles per cell",
            "api": "xclim_b200.calendar.percentile_doy + xclim_b200.indices.tx90p(bootstrap=True), device-resident Fields",
            "value": cells_total / (ms * 1e-3), "unit": "grid-cells/s", "ms_per_step": ms, "ms_bootstrap_kernel": ms_k,
            "steps": bsteps,
            "roofline": roofline(ctx, alg, ms_k, "bootstrap5_kernel<GT>", [T, ctx.rows, X], bound="compute (min/max pipe); "
                                 "fraction of the HBM roofline reported for reference"),
            "cpu_baseline": {"value": sel_b.size / dt, "unit": "grid-cells/s", "cores": 1, "kind": "port",
                             "sample": f"(10950, {sel_b.size}) cells, literal bootstrap restatement, {dt:.1f} s"},
            "check": {"oracle_cells_per_rank": int(sel_b.size), "bootstrap_bit_exact": boot_equal},
        }
        del res, got, fld, base
    del tasmax
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ fire weather
def fwi_section(ctx, rows=93):
    """SURVEY 8(f).4: the six Canadian Fire Weather Index System indices (cffwis_indices, always-on season) on a
    lat band of the grid, device-resident, with a sampled-cell check against the oracle.  It runs last and
    guarded.  A lane walks its cell through all T days, so the time of a launch is a whole number of waves of
    resident threads: on an H100 SXM 93 rows = 1,047 CTAs = 0.99 waves of the 1,056 CTAs that fit (8 per SM at
    64 registers, 132 SMs).  Two waves (187 rows) would need 118 GB for the four inputs and six outputs."""
    import torch
    from oracle import fire_oracle as FO
    from xclim_b200 import device, fire
    T, X = T_FULL, X_FULL
    rows = min(rows, ctx.rows)
    C = rows * X
    steps = max(1, min(ctx.args.steps, 3))
    kw = dict(cells_per_lat=X, n_lat_global=ctx.n_lat_global, cell_offset=ctx.row0 * X)
    tas = device.synth(T, C, kind=1, seed=3, **kw)
    tas.sub_(273.15)                                        # degC
    pr = device.synth(T, C, kind=0, seed=2, **kw)           # mm/d
    hurs = device.synth(T, C, kind=1, seed=11, **kw)
    hurs.sub_(hurs.mean()).mul_(4.0).add_(55.0).clamp_(5.0, 100.0)   # %
    ws = device.synth(T, C, kind=1, seed=12, **kw)
    ws.sub_(270.0).abs_().mul_(0.5)                         # km/h
    month = (np.minimum((np.arange(T) % YEAR) // 30.42, 11) + 1).astype(np.int8)
    lat_rows = np.linspace(-90.0, 90.0, ctx.n_lat_global)[ctx.row0:ctx.row0 + rows]
    lat = np.repeat(lat_rows, X)
    lat_d = torch.from_numpy(lat).to(ctx.dev)              # resident: no host copy inside the timed calls
    p = {k: (v if not isinstance(v, tuple) else v[0]) for k, v in fire.default_params.items()}
    P = device.fwi_params(None, False, None, True, **p)
    outs = ["DC", "DMC", "FFMC", "ISI", "BUI", "FWI"]
    run = lambda: device.fire_weather(tas, pr, hurs, ws, None, month, lat_d, None, None, None, None, None, outs, P)  # noqa: E731
    ms = timeit(ctx, run, steps, warmup=1)                  # the outputs of a call are released before the next one
    res = run()
    torch.cuda.synchronize()
    # sampled cells against the oracle (the same float32 series, copied back)
    sel = sample_cells(C, 48, 23 + ctx.rank)
    idx = torch.from_numpy(sel).to(ctx.dev)
    host = [x[:, idx].cpu().numpy() for x in (tas, pr, hurs, ws)]
    nanv = np.full(sel.size, np.nan, np.float32)
    t0 = time.perf_counter()
    exp = FO.fire_weather_calc(host[0], host[1], host[2], host[3], None, month, lat[sel], None, nanv, nanv, nanv,
                               np.zeros(sel.size, np.float32), outputs=outs)
    dt = time.perf_counter() - t0
    worst = {}
    for k in outs:
        got = res[k][:, idx].cpu().numpy().astype(np.float64)
        e = exp[k].astype(np.float64)
        with np.errstate(all="ignore"):
            rel = np.abs(got - e) / np.maximum(np.abs(e), 1e-3)
            if k == "FWI":   # Eq. 30b (fwi -> exp(2.72 (0.434 ln fwi)^0.647), fwi > 1) amplifies a difference of its input:
                ln_in = (np.log(e) / 2.72) ** (1.0 / 0.647) / 0.434          # errors are reported per unit of its
                cond = 2.72 * 0.647 * 0.434 ** 0.647 * ln_in ** -0.353       # condition number (unbounded at fwi = 1)
                rel = rel / np.where(e > 1.0, np.clip(np.nan_to_num(cond, nan=1.0, posinf=200.0), 1.0, 200.0), 1.0)
        rel = np.where(np.isnan(e) & np.isnan(got), 0.0, rel)
        worst[k] = float(np.nanmax(rel)) if np.isfinite(rel).all() else float("inf")
    ok = all(v <= 1e-5 for v in worst.values())
    alg = (4 + len(outs)) * T * C * 4
    r = roofline(ctx, alg, ms, "fwi_kernel<false>", None)
    r["bound"] = "FP64 pipe expected (about twenty float64 transcendentals per element); fraction of the HBM roofline reported"
    del res
    return {
        "workload": f"cffwis_indices (DC, DMC, FFMC, ISI, BUI, FWI; season always on) on a ({T},{rows},{X}) f32 band: "
                    "tas degC, pr mm/d, hurs %, sfcWind km/h; device-resident",
        "value": C / (ms * 1e-3), "unit": "grid-cells/s", "ms_per_step": ms, "steps": steps, "gpu_launches_per_step": 1,
        "roofline": r,
        "cpu_baseline": {"value": sel.size / dt, "unit": "grid-cells/s", "cores": 1, "kind": "port",
                         "sample": f"({T}, {sel.size}) cells, oracle day loop, {dt:.1f} s"},
        "check": {"oracle_cells": int(sel.size), "max_rel_err": worst, "tolerance": 1e-5, "within_tolerance": bool(ok),
                  "note": "FWI errors are divided by the condition number of Eq. 30b where it exceeds 1"},
    }


# ------------------------------------------------------------------------------------------------ EQM
def eqm_section(ctx):
    """EmpiricalQuantileMapping train + adjust.  ref, hist and the adjusted output of the full grid are 136 GB: a
    rank whose tile does not fit runs it on lat sub-tiles one after the other (inputs regenerated between
    sub-tiles, outside the timed regions) and the times add up."""
    import torch
    from oracle import xclim_oracle as O
    from xclim_b200 import device
    args = ctx.args
    T, X = T_FULL, X_FULL
    nq = 20
    steps = max(1, min(args.steps, 3))
    free, _ = torch.cuda.mem_get_info()
    per_row = 3 * T * X * 4                          # ref, hist (adjusted in place into sim), scen
    max_rows = int((free * 0.85 - (2 << 30)) // (per_row * 1.05))
    n_sub = max(1, -(-ctx.rows // max(1, max_rows)))
    bounds = np.linspace(0, ctx.rows, n_sub + 1).astype(int)
    ms_train = ms_adj = dt = 0.0
    err_af = err_sc = 0.0
    n_checked = 0
    for si in range(n_sub):
        rows = int(bounds[si + 1] - bounds[si])
        row0 = ctx.row0 + int(bounds[si])
        Cs = rows * X
        gen = lambda kind, seed: device.synth(T, Cs, kind=kind, seed=seed, cell_offset=row0 * X, cells_per_lat=X,  # noqa: E731
                                              n_lat_global=ctx.n_lat_global)
        ref = gen(1, 4)
        hist = gen(1, 5)
        hist.mul_(1.2).add_(1.5 - 0.2 * 288.0)          # +1.5 K bias, x1.2 variance about 288 K
        ms_train += timeit(ctx, lambda: device.eqm_train(ref, hist, nq, 0), steps, warmup=1)
        af, hq = device.eqm_train(ref, hist, nq, 0)
        if si == 0:
            sel = sample_cells(Cs, 32, 31 + ctx.rank)
            idx = torch.from_numpy(sel).to(ctx.dev)
            rs, hs = ref[:, idx].cpu().numpy(), hist[:, idx].cpu().numpy()
        del ref
        torch.cuda.empty_cache()
        sim = hist                                       # sim = hist-like + 2 K trend, built in place
        trend = torch.linspace(0.0, 2.0, T, device=ctx.dev, dtype=torch.float32)[:, None]
        sim.add_(trend)
        ms_adj += timeit(ctx, lambda: device.eqm_adjust(sim, af, hq, 0, 1), steps, warmup=1)
        scen = device.eqm_adjust(sim, af, hq, 0, 1)
        if si == 0:
            ss = sim[:, idx].cpu().numpy()
            t0 = time.perf_counter()
            af_o, hq_o = O.eqm_train(rs, hs, nq, "+")
            sc_o = O.eqm_adjust(ss, af_o, hq_o, "+", "linear")
            dt = time.perf_counter() - t0
            err_af = float(np.nanmax(np.abs(af[:, idx].cpu().numpy() - af_o) / np.maximum(np.abs(af_o), 1.0)))
            err_sc = float(np.nanmax(np.abs(scen[:, idx].cpu().numpy() - sc_o) / np.abs(sc_o)))
            assert err_sc < 1e-5 and err_af < 1e-4, (err_af, err_sc)
            n_checked = int(sel.size)
        del sim, hist, scen, af, hq
        torch.cuda.empty_cache()
    C = ctx.rows * X
    alg = 2 * T * C * 4 + 2 * nq * C * 4
    cells_total = ctx.n_lat_global * X
    tile = [T, ctx.rows, X] if n_sub == 1 else None
    return {
        "workload": f"EmpiricalQuantileMapping train(ref, hist, nquantiles={nq}, kind='+', group='time') + "
                    f"adjust(sim, interp='linear', extrapolation='constant') on ({T},{ctx.n_lat_global},{X}) f32, "
                    f"lat-tiled over {ctx.world} rank(s)",
        "value": cells_total / ((ms_train + ms_adj) * 1e-3), "unit": "grid-cells/s", "ms_train": ms_train,
        "ms_adjust": ms_adj, "steps": steps, "lat_subtiles_per_rank": int(n_sub),
        "roofline_train": roofline(ctx, alg, ms_train, "eqm_train_group_kernel<32 cells per CTA> (xc_eqm_train_f32 default dispatch)", tile),
        "roofline_adjust": roofline(ctx, alg, ms_adj, "eqm_adjust_kernel", tile),
        "cpu_baseline": {"value": n_checked / dt if dt else None, "unit": "grid-cells/s", "cores": 1, "kind": "port",
                         "sample": f"(10950, {n_checked}) cells, train + adjust restatement, {dt:.2f} s"},
        "check": {"oracle_cells_per_rank": n_checked, "max_rel_err_af": err_af, "max_rel_err_scen": err_sc,
                  "tolerance": 1e-5,
                  "parity": "unpinned: xsdba is not installed; compared with the oracle restatement only"},
    }


# ------------------------------------------------------------------------------------------------ batch of 50
def batch50_section(ctx):
    """BASELINE configs[4]: 50 indicators over tas / tasmax / tasmin / pr.  Four variables of the full grid are
    182 GB: a rank whose tile does not fit runs the batch on lat sub-tiles one after the other (inputs
    regenerated between sub-tiles, outside the timed regions) and the times add up."""
    import torch
    import xclim_b200
    from oracle import batch50 as OB
    from oracle import xclim_oracle as O
    from xclim_b200 import Field, TimeAxis, calendar as xcal, indices
    args = ctx.args
    T, X = T_FULL, X_FULL
    free, total = torch.cuda.mem_get_info()
    per_row = 4 * T * X * 4
    max_rows = int((free * 0.80 - (8 << 30)) // (per_row * 1.12))
    n_sub = max(1, -(-ctx.rows // max(1, max_rows)))
    bounds = np.linspace(0, ctx.rows, n_sub + 1).astype(int)
    ta = TimeAxis.daily("1981-01-01", T, "noleap")
    steps = max(1, min(args.steps, 2))
    tot_ms, launches, out_bytes, checked = 0.0, 0, 0, []
    cpu_dt, cpu_cells = 0.0, 0
    for si in range(n_sub):
        rows = int(bounds[si + 1] - bounds[si])
        row0 = ctx.row0 + int(bounds[si])
        Cs = rows * X
        from xclim_b200 import device
        gen = lambda kind, seed: device.synth(T, Cs, kind=kind, seed=seed, cell_offset=row0 * X, cells_per_lat=X,  # noqa: E731
                                              n_lat_global=ctx.n_lat_global)
        tasmax = gen(1, 3)
        tasmin = gen(1, 8)
        tasmin.sub_(8.0)
        tas = torch.add(tasmax, tasmin).mul_(0.5)
        pr = gen(0, 2)
        mk = lambda t, u: Field(t.view(T, rows, X), ("time", "lat", "lon"), ta, {}, {"units": u})  # noqa: E731
        fields = {"tas": mk(tas, "K"), "tasmax": mk(tasmax, "K"), "tasmin": mk(tasmin, "K"), "pr": mk(pr, "mm/d")}
        with xclim_b200.set_options(device_outputs=True):
            pers = {("tasmax", 90.0): None, ("tasmax", 10.0): None, ("tasmin", 90.0): None}
            for (var, p_) in list(pers):
                pers[(var, p_)] = xcal.select_percentile(xcal.percentile_doy(fields[var], window=5, per=p_), p_)
        per_of = {"tx90p": ("tasmax", 90.0), "tx10p": ("tasmax", 10.0), "tn90p": ("tasmin", 90.0)}

        def run_batch():
            outs = {}
            with xclim_b200.set_options(device_outputs=True):
                if hasattr(indices, "run_batch"):
                    return indices.run_batch(fields, pers=pers)
                for name, var in indices.BATCH_INDICATORS:
                    fn = getattr(indices, name)
                    outs[name] = fn(fields[var], pers[per_of[name]]) if name in per_of else fn(fields[var])
            return outs

        outs = run_batch()
        torch.cuda.synchronize()
        ctx.barrier()
        t0 = time.perf_counter()
        for _ in range(steps):
            outs = run_batch()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3 / steps
        tot_ms += ms
        out_bytes += sum(int(np.prod(o.values.shape)) * o.values.element_size() for o in outs.values())
        # sampled-cell check of every indicator against its oracle composition
        if si == 0:
            sel = sample_cells(Cs, 8, 41 + ctx.rank)[:24]
            idx = torch.from_numpy(sel).to(ctx.dev)
            host = {k: f.values.reshape(T, Cs)[:, idx].cpu().numpy() for k, f in fields.items()}
            import inspect
            t0 = time.perf_counter()
            for name, var in indices.BATCH_INDICATORS:
                x = host[var]
                freq = inspect.signature(getattr(indices, name)).parameters["freq"].default
                poff = ta.period_offsets(freq)
                got = outs[name].values.reshape(len(poff) - 1, Cs)[:, idx].cpu().numpy()
                if name in per_of:
                    p_ = per_of[name][1]
                    tab = O.percentile_doy(x, ta.year, ta.doy, 5, p_)[:, 0]
                    exp = O.doy_threshold_count(x, tab, ta.doy, poff, "<" if name == "tx10p" else ">")
                else:
                    exp = np.asarray(OB.oracle_indicator(name, x, poff))
                np.testing.assert_allclose(got, exp, rtol=1e-5, atol=1e-6, equal_nan=True, err_msg=name)
                checked.append(name)
            cpu_dt, cpu_cells = time.perf_counter() - t0, sel.size
        del outs, fields, pers, tas, tasmax, tasmin, pr
        torch.cuda.empty_cache()
    (tot_ms,) = ctx.max_over_ranks([tot_ms])
    C = ctx.rows * X
    cells_total = ctx.n_lat_global * X
    unique = 4 * T * C * 4 + 3 * YEAR * C * 8
    summed = 50 * T * C * 4
    r = roofline(ctx, unique + out_bytes, tot_ms, "batch of 50 (unique input bytes once + outputs)")
    r["effective_gbs_summed_inputs"] = summed / (tot_ms * 1e-3) / 1e9
    r["traffic_ratio_if_unfused"] = summed / unique
    return {
        "workload": f"50 atmos-style indices (xclim_b200.indices.BATCH_INDICATORS) over tas/tasmax/tasmin/pr "
                    f"({T},{ctx.n_lat_global},{X}) f32, lat-tiled over {ctx.world} rank(s), device-resident inputs and outputs",
        "value": cells_total / (tot_ms * 1e-3), "unit": "grid-cells/s", "ms_per_step": tot_ms, "steps": steps,
        "lat_subtiles_per_rank": int(n_sub), "timer": "host perf_counter around the batch, cuda synchronize both sides, "
                                                      "max over ranks (includes the Python launch overhead)",
        "roofline": r,
        "cpu_baseline": {"value": cpu_cells / cpu_dt if cpu_dt else None, "unit": "grid-cells/s", "cores": 1,
                         "kind": "port", "sample": f"(10950, {cpu_cells}) cells, 50 oracle compositions, {cpu_dt:.1f} s"},
        "check": {"indicators_checked": len(checked), "oracle_cells": int(cpu_cells), "tolerance": "exact for counts / "
                  "spells, 1e-5 for float reductions"},
    }


# ------------------------------------------------------------------------------------------------ e2e
def _bind_to_gpu_numa_node(local_index: int) -> str:
    """Pin this process (and therefore the first-touch placement of its pinned host buffer) to the CPUs
    of the NUMA node the GPU hangs off, so that H2D DMA reads local memory when 8 ranks stream at once.
    Best effort: any failure leaves the affinity untouched.  Disable with XCLIM_B200_NO_NUMA=1."""
    if os.environ.get("XCLIM_B200_NO_NUMA"):
        return "disabled"
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(local_index)
        bus = pynvml.nvmlDeviceGetPciInfo(h).busId
        bus = bus.decode() if isinstance(bus, bytes) else bus
        bus = bus.lower()
        if len(bus.split(":")[0]) == 8:      # nvml prints an 8-digit domain, sysfs uses 4
            bus = bus[4:]
        node = int(open(f"/sys/bus/pci/devices/{bus}/numa_node").read().strip())
        if node < 0:
            return "no numa info"
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.update(range(int(a), int(b or a) + 1))
        allowed = os.sched_getaffinity(0) & cpus
        if not allowed:
            return "no allowed cpu on node"
        os.sched_setaffinity(0, allowed)
        return f"node {node} ({len(allowed)} cpus)"
    except Exception as e:  # pragma: no cover - depends on the host
        return f"unavailable ({type(e).__name__})"


def e2e_section(ctx, pr_dev, poff, ref_out, ref_valid):
    """The headline metric end to end through the Python index function a user calls:
    ``xclim_b200.atmos.maximum_consecutive_dry_days(Field(host numpy array))`` -- host (pinned) input, lat slabs
    streamed H2D inside the call (xclim_b200.streaming), kernels per slab, results copied back to a numpy
    array.  The second leg runs tx90p the same way (percentile_doy + tx90p, two streamed calls)."""
    import torch
    from xclim_b200 import Field, TimeAxis, atmos, calendar as xcal, indices
    args = ctx.args
    T, C = pr_dev.shape
    X = X_FULL
    P = len(poff) - 1
    numa = _bind_to_gpu_numa_node(ctx.dev.index if ctx.dev.index is not None else 0)
    try:
        x_host = torch.empty((T, ctx.rows, X), dtype=torch.float32, pin_memory=True)
    except RuntimeError as e:  # not enough lockable host memory
        return {"value": None, "unit": "grid-cells/s", "error": f"cannot pin {T * C * 4 / 1e9:.1f} GB: {e}"}
    xh2 = x_host.view(T, C)
    for s in range(0, T, YEAR):
        xh2[s:s + YEAR].copy_(pr_dev[s:s + YEAR], non_blocking=True)
    torch.cuda.synchronize()
    ta = TimeAxis.daily("1981-01-01", T, "noleap")
    fld = Field(x_host.numpy(), ("time", "lat", "lon"), ta, {}, {"units": "mm/d"})
    call = lambda: atmos.maximum_consecutive_dry_days(fld, thresh="1 mm/day", freq="YS")  # noqa: E731
    res = call()
    for _ in range(2):
        res = call()
    exp = ref_out.clone()
    exp[ref_valid != YEAR] = float("nan")
    assert isinstance(res.values, np.ndarray) and res.values.shape == (P, ctx.rows, X)
    assert np.array_equal(res.values.reshape(P, C), exp.cpu().numpy(), equal_nan=True), \
        "e2e result differs from the device-resident result"
    steps = max(1, min(args.steps, 5))
    ctx.barrier()
    t0 = time.perf_counter()
    for _ in range(steps):
        call()
    ctx.barrier()
    (dt,) = ctx.max_over_ranks([(time.perf_counter() - t0) / steps])
    h2d = T * C * 4
    d2h = P * C * 4
    cells_total = ctx.n_lat_global * X
    out = {"value": cells_total / dt, "unit": "grid-cells/s", "ms_per_step": dt * 1e3, "steps": steps,
           "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h, "h2d_gbs_per_rank": h2d / dt / 1e9,
           "api": "xclim_b200.atmos.maximum_consecutive_dry_days(Field(numpy (time, lat, lon) f32, pinned host memory)) "
                  "-> numpy (periods, lat, lon) f32 with MissingAny NaNs; lat slabs streamed H2D on a copy stream "
                  "while the kernels of the previous slab run (xclim_b200/streaming.py)",
           "numa_binding": numa,
           "timer": "host perf_counter around the synchronous calls, barrier + cuda sync both sides, max over ranks"}
    del fld, x_host, xh2
    # ---- tx90p end to end (two streamed calls: percentile_doy, then the count against the host table)
    if "tx90p" in args.sections:
        try:
            th = torch.empty((T, ctx.rows, X), dtype=torch.float32, pin_memory=True)
        except RuntimeError as e:
            out["tx90p"] = {"error": str(e)}
            return out
        from xclim_b200 import device
        th2 = th.view(T, C)
        band = 16 * X     # the tile's tasmax is generated in bands of 16 rows: the headline input is still resident
        for c0 in range(0, C, band):
            c1 = min(C, c0 + band)
            tdev = device.synth(T, c1 - c0, kind=1, seed=3, cell_offset=ctx.row0 * X + c0, cells_per_lat=X,
                                n_lat_global=ctx.n_lat_global)
            th2[:, c0:c1].copy_(tdev)
            del tdev
        torch.cuda.empty_cache()
        tf = Field(th.numpy(), ("time", "lat", "lon"), ta, {}, {"units": "K"})

        def call_tx():
            per = xcal.select_percentile(xcal.percentile_doy(tf, window=5, per=90.0), 90.0)
            return indices.tx90p(tf, per, freq="YS")

        r = call_tx()
        frac = float(np.mean(r.values)) / YEAR
        assert 0.07 < frac < 0.13, frac
        n2 = max(1, min(args.steps, 2))
        ctx.barrier()
        t0 = time.perf_counter()
        for _ in range(n2):
            call_tx()
        ctx.barrier()
        (dt2,) = ctx.max_over_ranks([(time.perf_counter() - t0) / n2])
        out["tx90p"] = {"value": cells_total / dt2, "unit": "grid-cells/s", "ms_per_step": dt2 * 1e3, "steps": n2,
                        "h2d_bytes_per_step": 2 * T * C * 4 + YEAR * C * 8, "d2h_bytes_per_step": YEAR * C * 8 + P * C * 8,
                        "api": "xclim_b200.calendar.percentile_doy(Field(numpy)) + xclim_b200.indices.tx90p(Field(numpy), per): "
                               "the input crosses PCIe twice (two calls, as in the reference API)"}
        del tf, th, th2
    return out
