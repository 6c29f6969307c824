#!/usr/bin/env python
"""Secondary measurements (not the driver's contract): BASELINE.json configs 3b (bootstrap) and 4 (EQM)
plus the other streaming kernels, on a lat band of the headline grid.  One JSON line per kernel.
With --cpu every line also carries `cpu_port`: the oracle restatement (numpy, the reference's
whole-array algorithm) of the same index timed on ONE host core over a small sample of the same
cells -- a baseline beside the kernel, never the thing measured.

    python bench_extra.py --lat 180 --steps 3
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
T, X, YEAR = 10950, 1440, 365


WARMUP = 2


def timeit(fn, steps, warmup=None):
    import torch
    warmup = WARMUP if warmup is None else min(warmup, WARMUP)
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    ev[0].record()
    for i in range(steps):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    return float(np.mean([ev[i].elapsed_time(ev[i + 1]) for i in range(steps)]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lat", type=int, default=180)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--only", default="")
    ap.add_argument("--warmup", type=int, default=2, help="untimed launches per kernel (0 for ncu captures)")
    ap.add_argument("--cpu", action="store_true", help="time the oracle port of every index on a cell sample")
    ap.add_argument("--cpu-cells", type=int, default=1024)
    a = ap.parse_args()
    global WARMUP
    WARMUP = a.warmup
    import torch
    from xclim_b200 import _lib, device
    C = a.lat * X
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))).get("hbm_gbs", 3350.0) \
        if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0
    poff = np.arange(T // YEAR + 1, dtype=np.int32) * YEAR
    poff_m = None
    doy = (np.arange(T) % YEAR + 1).astype(np.int16)
    yidx = (np.arange(T) // YEAR).astype(np.int16)
    tas = device.synth(T, C, kind=1, seed=3, cells_per_lat=X, n_lat_global=a.lat)
    pr = device.synth(T, C, kind=0, seed=2, cells_per_lat=X, n_lat_global=a.lat)

    S = a.cpu_cells
    O = None
    host = {}
    if a.cpu:
        from oracle import xclim_oracle as O  # noqa: N811  (CPU baseline leg only)
        host = {"tas": tas[:, :S].cpu().numpy(), "pr": pr[:, :S].cpu().numpy()}

    def report(name, ms, alg_bytes, extra=None, cpu=None, cpu_cells=None):
        gbs = alg_bytes / (ms * 1e-3) / 1e9
        line = {"kernel": name, "grid": [T, a.lat, X], "ms": ms, "cells_per_s": C / (ms * 1e-3),
                "algorithmic_bytes": alg_bytes, "achieved_gbs": gbs, "frac_of_measured_hbm_peak": gbs / peak}
        if extra:
            line.update(extra)
        if a.cpu and cpu is not None:
            import time
            n = cpu_cells or S
            t0 = time.perf_counter()
            cpu()
            dt = time.perf_counter() - t0
            line["cpu_port"] = {"value": n / dt, "unit": "grid-cells/s", "cores": 1, "kind": "port",
                                "sample": f"({T}, {n}) cells, {dt:.2f} s"}
            line["gpu_over_one_core"] = line["cells_per_s"] / (n / dt)
        print(json.dumps(line), flush=True)

    want = lambda k: (not a.only) or (k in a.only.split(","))
    P = T // YEAR
    if want("count"):
        ms = timeit(lambda: device.period_count(pr, poff, _lib.OPS[">="], 1.0, want_valid=True), a.steps)
        report("period_count (wetdays, fused valid)", ms, T * C * 4 + 2 * P * C * 4,
               cpu=lambda: O.threshold_count(host["pr"], ">=", 1.0, poff))
    if want("reduce"):
        ms = timeit(lambda: device.period_reduce(tas, poff, _lib.STATS["mean"], want_valid=True), a.steps)
        report("period_reduce mean (tg_mean, fused valid)", ms, T * C * 4 + 2 * P * C * 4,
               cpu=lambda: O.select_resample_op(host["tas"], "mean", poff))
    if want("runsum"):
        ms = timeit(lambda: device.period_runstat(pr, poff, _lib.OPS["<"], 1.0, _lib.RL_REDUCERS["sum"], 3), a.steps)
        report("period_runstat sum window=3 (windowed_run_count)", ms, T * C * 4 + P * C * 4,
               cpu=lambda: O.resample_and_rl(O.compare(host["pr"], "<", 1.0), True, O.rle_statistics, poff=poff,
                                             reducer="sum", window=3))
    if want("after"):
        ms = timeit(lambda: device.period_runstat(pr, poff, _lib.OPS["<"], 1.0, _lib.RL_REDUCERS["max"], 1, False),
                    a.steps)
        report("period_runstat max, resample_before_rl=False", ms, T * C * 4 + P * C * 4,
               cpu=lambda: O.resample_and_rl(O.compare(host["pr"], "<", 1.0), False, O.rle_statistics, poff=poff,
                                             reducer="max", window=1))
    if want("rolling"):
        ms = timeit(lambda: device.rolling_period_reduce(pr, poff, 5, _lib.STATS["sum"], False, _lib.STATS["max"]),
                    a.steps)
        report("rolling(5).sum -> max (max_n_day_precipitation_amount)", ms, T * C * 4 + P * C * 4,
               cpu=lambda: O.select_rolling_resample_op(host["pr"], "max", 5, poff, window_center=False,
                                                        window_op="sum"))
    if want("spell"):
        ms = timeit(lambda: device.spell_runstat(pr, poff, 3, _lib.STATS["sum"], _lib.OPS["<"], 1.0,
                                                 _lib.RL_REDUCERS["count"]), a.steps)
        report("spell_runstat window=3 sum<1 count (dry_spell_frequency)", ms, T * C * 4 + P * C * 4,
               cpu=lambda: O.spell_length_statistics(host["pr"], 1.0, 3, "sum", "<", "count", poff))
    if want("spellmean"):
        ms = timeit(lambda: device.spell_runstat(pr, poff, 3, _lib.STATS["sum"], _lib.OPS["<"], 1.0,
                                                 _lib.RL_REDUCERS["mean"]), a.steps)
        report("spell_runstat window=3 sum<1 mean (any-reducer spell_sumw_kernel)", ms, T * C * 4 + P * C * 4,
               cpu=lambda: O.spell_length_statistics(host["pr"], 1.0, 3, "sum", "<", "mean", poff))
    if want("spellmin"):
        ms = timeit(lambda: device.spell_runstat(tas, poff, 5, _lib.STATS["min"], _lib.OPS[">"], 291.15,
                                                 _lib.RL_REDUCERS["max"]), a.steps)
        report("spell_runstat window=5 min>291.15 max (spell_runstat4_kernel)", ms, T * C * 4 + P * C * 4,
               cpu=lambda: O.spell_length_statistics(host["tas"], 291.15, 5, "min", ">", "max", poff))
    if want("spell10"):   # a window past the register kernels' 2..8: the ring's sliding float64 sum
        ms = timeit(lambda: device.spell_runstat(pr, poff, 10, _lib.STATS["sum"], _lib.OPS["<"], 1.0,
                                                 _lib.RL_REDUCERS["count"]), a.steps)
        report("spell_runstat window=10 sum<1 count (spell_runstat4_kernel, sliding sum)", ms, T * C * 4 + P * C * 4,
               cpu=lambda: O.spell_length_statistics(host["pr"], 1.0, 10, "sum", "<", "count", poff))
    if want("rolling1"):
        ms = timeit(lambda: device.rolling_period_reduce(pr, poff, 1, _lib.STATS["sum"], False, _lib.STATS["min"]),
                    a.steps)
        report("rolling(1).sum -> min (rolling_period_reduce4_kernel, sliding sum)", ms, T * C * 4 + P * C * 4,
               cpu=lambda: O.select_rolling_resample_op(host["pr"], "min", 1, poff, window_center=False,
                                                        window_op="sum"))
    if want("gap"):
        ms = timeit(lambda: device.period_runstat_gap(pr, poff, _lib.OPS["<"], 1.0, _lib.RL_REDUCERS["max"], 3),
                    a.steps)
        report("period_runstat_gap min_gap=3 <1 max (spell_length_statistics min_gap)", ms, T * C * 4 + P * C * 4,
               cpu=lambda: O.spell_length_statistics(host["pr"], 1.0, 1, None, "<", "max", poff, min_gap=3))
    if want("first"):
        ms = timeit(lambda: device.period_boundary_run(tas, poff, _lib.OPS[">"], 283.15, 5), a.steps)
        report("period_boundary_run first, window=5", ms, T * C * 4 + P * C * 4,
               cpu=lambda: O.first_run(O.compare(host["tas"], ">", 283.15), 5, poff=poff))
    if want("heatwave"):
        tmin = tas - 8.0
        ms = timeit(lambda: device.period_runstat2(tmin, tas, poff, _lib.OPS[">"], 283.15, _lib.OPS[">"], 291.15,
                                                   _lib.RL_REDUCERS["count"], 3), a.steps)
        report("period_runstat2 (heat_wave_frequency: tasmin & tasmax, window 3)", ms, 2 * T * C * 4 + P * C * 4,
               cpu=lambda: O.resample_and_rl(O.compare(host["tas"] - np.float32(8.0), ">", 283.15)
                                             & O.compare(host["tas"], ">", 291.15), True, O.rle_statistics, poff=poff,
                                             reducer="count", window=3))
        del tmin
    if want("maxsum"):
        ms = timeit(lambda: device.period_run_maxsum(tas, poff, _lib.OPS[">"], 291.15, 3), a.steps)
        report("period_run_maxsum (hot_spell_max_magnitude, window 3)", ms, T * C * 4 + P * C * 4,
               cpu=lambda: O.resample_and_rl(np.clip(host["tas"] - np.float32(291.15), 0, None).astype(np.float64),
                                             True, O.windowed_max_run_sum, 3, poff=poff))
    if want("runq"):
        ms = timeit(lambda: device.period_run_quantile(pr, poff, _lib.OPS["<"], 1.0, 0.9, 1), a.steps)
        report("period_run_quantile q90 of dry-run lengths (rle_statistics reducer='q90')", ms, T * C * 4 + P * C * 4)
    if want("doycount"):
        tab = device.percentile_doy(tas, doy, yidx, YEAR, P, 5, [90.0], 1 / 3, 1 / 3)[0]
        poff_ms = np.concatenate([[0], np.cumsum(np.tile([31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31], P))]).astype(np.int32)
        ms = timeit(lambda: device.doy_threshold_count(tas, poff_ms, doy, tab, _lib.OPS[">"]), a.steps)
        report("period_count_thr_kernel (tx90p count, freq=MS: generic periods)", ms,
               T * C * 4 + YEAR * C * 8 + (len(poff_ms) - 1) * C * 4)
        del tab
    if want("bootstrap"):
        nb = 15
        step_period = np.repeat(np.arange(nb), YEAR).astype(np.int32)
        fn = lambda: device.bootstrap_doy_count(tas, 0, nb, YEAR, step_period, P, 5, 90.0, 1 / 3, 1 / 3, _lib.OPS[">"])
        ms = timeit(fn, max(1, a.steps // 2), warmup=1)
        yr_full = (np.arange(T) // YEAR).astype(np.int64)
        report("bootstrap_doy_count (tx90p 3b: 15-year base, 14 resamples per year)", ms, T * C * 4 + P * C * 8,
               {"quantile_evaluations_per_cell": nb * (nb - 1) * YEAR},
               cpu=lambda: O.bootstrap_doy_count(host["tas"][:, :4], yr_full, doy.astype(np.int64), poff, (0, nb - 1),
                                                 window=5, per=90.0, op=">"), cpu_cells=4)
    if want("batch50"):
        from xclim_b200 import Field, TimeAxis, indices, calendar as xcal
        ta = TimeAxis.daily("1981-01-01", T, "noleap")
        tasmin = tas - 8.0
        mk = lambda t, u: Field(t.reshape(T, a.lat, X), ("time", "lat", "lon"), ta, {}, {"units": u})  # noqa: E731
        fields = {"tas": mk(tas, "K"), "tasmax": mk(tas, "K"), "tasmin": mk(tasmin, "K"), "pr": mk(pr, "mm/d")}
        pers = {p_: xcal.select_percentile(xcal.percentile_doy(fields["tasmax"], window=5, per=p_), p_) for p_ in (10.0, 90.0)}

        def run_batch():
            for name, var in indices.BATCH_INDICATORS:
                fn = getattr(indices, name)
                if name in ("tx90p", "tn90p"):
                    fn(fields[var], pers[90.0])
                elif name == "tx10p":
                    fn(fields[var], pers[10.0])
                else:
                    fn(fields[var])
        import time
        import xclim_b200
        for dev_out in (False, True):
            with xclim_b200.set_options(device_outputs=dev_out):
                run_batch()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                run_batch()
                torch.cuda.synchronize()
                ms = (time.perf_counter() - t0) * 1e3
            report("batch of 50 atmos indicators (sequential calls, outputs "
                   + ("left in HBM: set_options(device_outputs=True))" if dev_out else "copied to host)"), ms,
                   50 * T * C * 4,
                   {"unique_input_bytes": 4 * T * C * 4,
                    "note": "effective GB/s = sum of per-indicator input bytes / time"})
    if want("eqm"):
        hist = device.synth(T, C, kind=1, seed=5, cells_per_lat=X, n_lat_global=a.lat)
        ms = timeit(lambda: device.eqm_train(tas, hist, 20, 0), max(1, a.steps // 2), warmup=1)
        if a.cpu:
            host["hist"] = hist[:, :S].cpu().numpy()
        report("eqm_train nq=20 (ref, hist)", ms, 2 * T * C * 4 + 2 * 20 * C * 4,
               cpu=lambda: O.eqm_train(host["tas"], host["hist"], 20, "+"))
        af, hq = device.eqm_train(tas, hist, 20, 0)
        ms = timeit(lambda: device.eqm_adjust(hist, af, hq, 0, 1), a.steps)
        if a.cpu:
            haf, hhq = O.eqm_train(host["tas"], host["hist"], 20, "+")
        report("eqm_adjust linear (sim -> scen)", ms, 2 * T * C * 4 + 2 * 20 * C * 4,
               cpu=lambda: O.eqm_adjust(host["hist"], haf, hhq, "+", "linear"))
    if want("qdm"):
        from xclim_b200.sdba import equally_spaced_nodes
        hist = af = hq = None      # the EQM section's buffers: sim, scen and sim_q need the room
        hist = device.synth(T, C, kind=1, seed=5, cells_per_lat=X, n_lat_global=a.lat)
        af, _ = device.eqm_train(tas, hist, 20, 0)
        nodes = equally_spaced_nodes(20).astype(np.float32)
        if a.cpu:
            from oracle import qdm_oracle as QO
            host["hist"] = hist[:, :S].cpu().numpy()
            qaf = af[:, :S].cpu().numpy()
        for with_q in (False, True):
            ms = timeit(lambda: device.qdm_adjust(hist, af, nodes, 0, 1, want_sim_q=with_q), a.steps)
            report("qdm_adjust linear nq=20 (sim -> scen" + (", sim_q float64)" if with_q else ")"), ms,
                   2 * T * C * 4 + 20 * C * 4 + (T * C * 8 if with_q else 0),
                   {"scratch_bytes_per_cell": 6 * T + 16},
                   cpu=lambda: QO.qdm_adjust(host["hist"], qaf, "+", "linear"))
    if want("dqm"):
        hist = af = hq = None
        hist = device.synth(T, C, kind=1, seed=5, cells_per_lat=X, n_lat_global=a.lat)
        if a.cpu:
            from oracle import dqm_oracle as DO
            host["hist"] = hist[:, :S].cpu().numpy()
        ms_mean = timeit(lambda: device.period_reduce(tas, [0, T], _lib.STATS["mean"]), a.steps)
        ms = timeit(lambda: device.dqm_train(tas, hist, 20, 0), a.steps)
        report("dqm_train nq=20 (means pass + selection on the normalised series)", ms, 2 * T * C * 4,
               {"means_pass_ms_each": ms_mean, "means_pass_algorithmic_bytes": 2 * T * C * 4},
               cpu=lambda: DO.dqm_train(host["tas"], host["hist"], 20, "+"))
        af, hq, sc = device.dqm_train(tas, hist, 20, 0)
        if a.cpu:
            daf, dhq, dsc = (v[..., :S].cpu().numpy() for v in (af, hq, sc))
        ms_fit = timeit(lambda: device.poly_fit(hist, 1, 0, sc), a.steps)
        ms = timeit(lambda: device.dqm_adjust(hist, af, hq, sc, 0, 1, 1), a.steps)
        report("dqm_adjust linear nq=20 detrend=1 (trend fit + apply, sim -> scen)", ms, 3 * T * C * 4,
               {"fit_ms": ms_fit},
               cpu=lambda: DO.dqm_adjust(host["hist"], daf, dhq, dsc, "+", "linear", detrend=1))
    if want("spi") and a.only:      # standardized precipitation index: opt-in (--only spi)
        from xclim_b200.timeaxis import TimeAxis
        ta = TimeAxis.daily("1981-01-01", T, "noleap")
        pm = ta.period_offsets("MS")
        Pm = pm.size - 1
        gid = (ta.month[pm[:-1]] - 1).astype(np.int64)
        order = np.argsort(gid, kind="stable")
        goff = np.concatenate([[0], np.cumsum(np.bincount(gid, minlength=12))])
        m, _ = device.period_reduce(pr, pm, _lib.STATS["mean"])
        r = device.rolling_mean(m, 3)
        prm, nz, nn, status = device.si_fit(r, goff, order, 0, 1, True, 0.0)
        ms_res = timeit(lambda: device.period_reduce(pr, pm, _lib.STATS["mean"]), a.steps)
        ms_roll = timeit(lambda: device.rolling_mean(m, 3), a.steps)
        ms_fit = timeit(lambda: device.si_fit(r, goff, order, 0, 1, True, 0.0), a.steps)
        ms_app = timeit(lambda: device.si_apply(r, gid, prm, nz, nn, 0), a.steps)
        # sampled cells, the last ones included: the kernel's parameters against the oracle's fit (kernel log rule)
        # and the kernel's index against the oracle's scipy transform of those parameters
        from oracle import stdindex_oracle as SO
        cols = np.unique(np.r_[np.linspace(0, C - 1, 48).astype(int), np.arange(C - 16, C)])
        rs, ps = r[:, cols].cpu().numpy(), prm[:, :, cols].cpu().numpy()
        po, _, _ = SO.fit_groups(rs, gid, 12, slice(None), "gamma", "ML", True, 0.0, numpy_logs=False)
        si = device.si_apply(r, gid, prm, nz, nn, 0)[:, cols].cpu().numpy()
        sio = SO.transform(rs, gid, ps, "gamma", nz[:, cols].cpu().numpy(), nn[:, cols].cpu().numpy())
        ok = ~np.isnan(sio)
        from scipy.stats import norm
        import subprocess
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True)
        card = {"gpu": torch.cuda.get_device_name(), "power_limit": q.stdout.strip() or "unknown"}
        check = {"cells": int(cols.size), "status": status, "nan_pattern_equal": bool(np.array_equal(np.isnan(si), ~ok)),
                 "max_shape_rel_diff": float(np.nanmax(np.abs(ps[:, 0] - po[:, 0]) / np.abs(po[:, 0]))),
                 "max_dsi_times_pdf": float(np.max(np.abs(si - sio)[ok] * norm.pdf(sio[ok])))}
        report("spi monthly SPI-3 gamma ML floc=0: resample + rolling + fit + apply", ms_res + ms_roll + ms_fit + ms_app,
               T * C * 4 + Pm * C * 4 + Pm * C * 4 + Pm * C * 8,
               {"resample_ms": ms_res, "resample_algorithmic_bytes": T * C * 4 + Pm * C * 4,
                "resample_gbs": (T * C * 4 + Pm * C * 4) / (ms_res * 1e-3) / 1e9, "rolling_ms": ms_roll,
                "fit_ms": ms_fit, "apply_ms": ms_app, "apply_elements_per_s": Pm * C / (ms_app * 1e-3),
                "apply_bound": "FP64 pipe: P(a, x) by series / continued fraction (tens of iterations) and two Halley "
                               "steps of the inverse normal per element",
                "check": check, **card})
        del m, r, prm, nz, nn
        Cd = min(a.lat, 90) * X                   # daily SPI-30 on a band: its float64 output is T * Cd * 8 bytes
        prd = pr[:, :Cd]
        gd = (ta.doy - 1).astype(np.int64)
        od = np.argsort(gd, kind="stable")
        gofd = np.concatenate([[0], np.cumsum(np.bincount(gd, minlength=365))])
        rd = device.rolling_mean(prd, 30)
        pd_, nzd, nnd, _ = device.si_fit(rd, gofd, od, 0, 1, True, 0.0)
        ms_roll = timeit(lambda: device.rolling_mean(prd, 30), a.steps)
        ms_fit = timeit(lambda: device.si_fit(rd, gofd, od, 0, 1, True, 0.0), a.steps)
        ms_app = timeit(lambda: device.si_apply(rd, gd, pd_, nzd, nnd, 0), a.steps)
        report(f"spi daily SPI-30 gamma ML floc=0 on {Cd // X} rows: rolling + fit + apply", ms_roll + ms_fit + ms_app,
               T * Cd * 4 * 2 + T * Cd * 8,
               {"rows": Cd // X, "rolling_ms": ms_roll, "fit_ms": ms_fit, "apply_ms": ms_app,
                "apply_elements_per_s": T * Cd / (ms_app * 1e-3), **card})
        del rd, pd_, nzd, nnd
    if want("evfit") and a.only:    # frequency analysis: opt-in (--only evfit), on its own full-grid maxima
        import subprocess
        from oracle import evfit_oracle as FO
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True)
        card = {"gpu": torch.cuda.get_device_name(), "power_limit": q.stdout.strip() or "unknown"}
        grid, band = 721 * X, 90 * X
        t_ret = np.array([2, 10, 20, 50, 100], np.float64)
        for P in (30, 150):
            # YS maxima of synthetic daily pr, made band by band (P years of daily data do not fit in HBM whole)
            poff_y = np.arange(P + 1, dtype=np.int32) * YEAR
            mx = torch.empty((P, grid), dtype=torch.float32, device="cuda")
            for c0 in range(0, grid, band):
                cb = min(band, grid - c0)
                d = device.synth(P * YEAR, cb, kind=0, seed=5, cell_offset=c0, cells_per_lat=X, n_lat_global=721)
                mx[:, c0:c0 + cb] = device.period_reduce(d, poff_y, _lib.STATS["max"])[0]
                del d
            for dist in ("genextreme", "gumbel_r"):
                code = _lib.EV_DISTS[dist]
                prm, status = device.ev_fit(mx, code)
                ms_fit = timeit(lambda: device.ev_fit(mx, code), a.steps)
                ms_tr = timeit(lambda: device.ev_transform(prm, code, _lib.EV_KINDS["isf"], 1.0 / t_ret), a.steps)
                rl = device.ev_transform(prm, code, _lib.EV_KINDS["isf"], 1.0 / t_ret)
                cols = np.unique(np.r_[np.linspace(0, grid - 1, 16).astype(int), np.arange(grid - 8, grid)])
                xs, ps, rls = mx[:, cols].cpu().numpy(), prm[:, cols].cpu().numpy(), rl[:, cols].cpu().numpy()
                worst_nnlf, worst_rl = 0.0, 0.0
                for k in range(cols.size):
                    po = FO.fit(xs[:, k], dist)
                    if dist == "genextreme":
                        fo = FO.gev_nnlf(po, xs[:, k])
                        worst_nnlf = max(worst_nnlf, (FO.gev_nnlf(ps[:, k], xs[:, k]) - fo) / max(1.0, abs(fo)))
                    ro = FO.return_levels(po[:, None], dist, t_ret)[:, 0]
                    worst_rl = max(worst_rl, float(np.max(np.abs(rls[:, k] - ro) / np.abs(ro))))
                nan_cells = int(torch.isnan(prm[0]).sum().item())
                report(f"evfit {dist} ML fit on YS maxima, P={P} x 721 x 1440 (+ isf at T=2..100)", ms_fit,
                       P * grid * 4 * 2 + prm.numel() * 8,
                       {"years": P, "fit_ms": ms_fit, "fit_cells_per_s": grid / (ms_fit * 1e-3),
                        "transform_ms": ms_tr, "transform_elements_per_s": t_ret.size * grid / (ms_tr * 1e-3),
                        "bound": "FP64 pipe: log1p / exp of every value in every Newton iteration",
                        "status": status, "nan_cells": nan_cells,
                        "oracle_check": {"cells": int(cols.size), "max_rel_nnlf_excess": worst_nnlf,
                                         "max_return_level_rel_diff": worst_rl}, **card})
                del prm, rl
            del mx
    if want("analog") and a.only:   # spatial analogues: opt-in (--only analog), one target against the full grid
        import subprocess
        from oracle import analog_oracle as AO
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True)
        card = {"gpu": torch.cuda.get_device_name(), "power_limit": q.stdout.strip() or "unknown"}
        grid, n, m, d = 721 * X, 30, 30, 3
        g = torch.Generator(device="cuda").manual_seed(17)
        shift = torch.randn((1, d, grid), generator=g, device="cuda")
        cand = (torch.randn((m, d, grid), generator=g, device="cuda") + shift).contiguous()
        tgt = cand[:, :, 1234].contiguous()[None].clone()                   # (1, n, d): one cell's own sample
        tx = tgt[0].double().cpu().numpy()
        cols = np.unique(np.r_[np.linspace(0, grid - 33, 224).astype(int), np.arange(grid - 32, grid)])
        ys = cand[:, :, cols].double().cpu().numpy()
        N, pairs = n + m, (n + m) * (n + m - 1) // 2
        # algorithmic float64 operations per cell (a sqrt or log counts as one): the pair loops dominate
        flops = {"seuclidean": 4 * N * d, "mahalanobis": 4 * N * d + 2 * d * d,
                 "zech_aslan": pairs * (4 * d + 2), "szekely_rizzo": pairs * (4 * d + 2),
                 "nearest_neighbor": N * (N - 1) * 3 * d, "kldiv": n * N * 3 * d + 2 * n,
                 "kolmogorov_smirnov": 0}
        for method, param in (("seuclidean", 0.0), ("nearest_neighbor", 0.0), ("zech_aslan", 1e-12),
                              ("szekely_rizzo", 1.0), ("kolmogorov_smirnov", 0.0), ("kldiv", 1.0),
                              ("mahalanobis", 0.0)):
            cst = AO.target_consts(tx, method)
            cst = None if cst is None else torch.from_numpy(np.asarray(cst).reshape(1, -1)).cuda()
            code = _lib.AN_METHODS[method]
            out, status = device.analog(tgt, cand, code, param, cst)
            ms = timeit(lambda: device.analog(tgt, cand, code, param, cst), a.steps)
            got = out[0, cols].cpu().numpy()
            kw = {"zech_aslan": {"dmin": param}, "kldiv": {"k": 1}}.get(method, {})
            ref = np.array([AO.metric(method, tx, ys[:, :, k], **kw) for k in range(cols.size)])
            worst = float(np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1e-300)))
            fl = flops[method] * grid
            extra = {"method": method, "cells": grid, "n": n, "m": m, "d": d, "status": status,
                     "fp64_ops": fl, "fp64_ops_per_s": fl / (ms * 1e-3),
                     "share_of_fp64_peak": fl / (ms * 1e-3) / 34e12,
                     "oracle_check": {"cells": int(cols.size), "max_rel_diff": worst}, **card}
            if method == "kolmogorov_smirnov":
                extra["comparisons"] = 2 * n * (2 * N * d + N * N) * grid
            report(f"analog {method}, n = m = 30, d = 3, 721 x 1440 cells", ms, cand.numel() * 4 + grid * 8, extra)
        del cand, shift
    if want("pet") and a.only:      # evapotranspiration: opt-in (--only pet), on the --lat band of the grid
        import subprocess
        from oracle import pet_oracle as PO
        from xclim_b200 import TimeAxis, converters
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True)
        card = {"gpu": torch.cuda.get_device_name(), "power_limit": q.stdout.strip() or "unknown"}
        ta = TimeAxis.daily("1981-01-01", T, "noleap")
        lat_u = np.linspace(-89.5, 89.5, a.lat)
        idx = np.repeat(np.arange(a.lat, dtype=np.int32), X)
        idx_d = torch.from_numpy(idx).cuda()
        cols = np.unique(np.r_[np.linspace(0, C - 1, 96).astype(int), np.arange(C - 32, C)])

        def params(method, wb, affine):
            P = _lib.PetParams()
            P.method, P.water_budget = _lib.PET_METHODS[method], int(wb)
            for i, name in enumerate(_lib.PET_INPUTS):
                P.in_scale[i], P.in_offset[i] = affine.get(name, (1.0, 0.0))
            P.wind_num, P.wind_den = float(np.log(67.8 * 2 - 5.42)), float(np.log(67.8 * 10 - 5.42))
            return P

        def ins(**kw):
            return [kw.get(n) for n in _lib.PET_INPUTS]

        def sample(x):
            return x[:, cols].cpu().numpy()

        tmin = tas - 5.0
        tmax = tas + 5.0
        degf = {"tasmin": (1.8, -459.67), "tasmax": (1.8, -459.67)}
        table = torch.from_numpy(converters._daily_table("BR65", ta, lat_u)).cuda()
        P = params("BR65", True, degf)
        out = device.pet_daily(ins(tasmin=tmin, tasmax=tmax, pr=pr), table, idx_d, P)
        ms = timeit(lambda: device.pet_daily(ins(tasmin=tmin, tasmax=tmax, pr=pr), table, idx_d, P), a.steps)
        f = lambda x: (x * np.float32(1.8) + np.float32(-459.67)).astype(np.float32)   # noqa: E731
        ref = np.float32(PO.daily_rate(PO.daily_pet("BR65", table.cpu().numpy()[:, idx[cols]], tasmin=f(sample(tmin)),
                                                    tasmax=f(sample(tmax))), sample(pr)))
        got = sample(out)
        report(f"pet BR65 water budget, {a.lat} x 1440 cells", ms, 4 * (3 + 1) * T * C,
               {"oracle_check": {"cells": int(cols.size), "bit_equal": bool(np.array_equal(got, ref, equal_nan=True))},
                **card})
        del out, table
        # FAO_PM98 on a 40-row band: eight input series
        C8 = 40 * X
        g = torch.Generator(device="cuda").manual_seed(5)
        ser = {k: (torch.rand((T, C8), generator=g, device="cuda") * s + o)
               for k, s, o in (("tasmin", 10, 270), ("tasmax", 10, 280), ("hurs", 0.9, 0.1), ("rsds", 300, 0),
                               ("rsus", 60, 0), ("rlds", 200, 200), ("rlus", 250, 200), ("sfcWind", 10, 0))}
        k2c = {"tasmin": (1.0, -273.15), "tasmax": (1.0, -273.15)}
        P = params("allen98", False, k2c)
        out = device.pet_daily(ins(**ser), None, None, P)
        ms = timeit(lambda: device.pet_daily(ins(**ser), None, None, P), a.steps)
        c8 = np.unique(np.r_[np.linspace(0, C8 - 1, 96).astype(int), np.arange(C8 - 32, C8)])
        sm = {k: v[:, c8].cpu().numpy() for k, v in ser.items()}
        for k in ("tasmin", "tasmax"):
            sm[k] = (sm[k] * np.float32(1.0) + np.float32(-273.15)).astype(np.float32)
        ref = np.float32(PO.daily_rate(PO.daily_pet("allen98", None, **sm)))
        got = out[:, c8].cpu().numpy()
        ulp = float(np.max(np.abs(got.view(np.int32).astype(np.int64) - ref.view(np.int32).astype(np.int64))))
        report("pet FAO_PM98, 40 x 1440 cells", ms, 4 * (8 + 1) * T * C8,
               {"cells": C8, "oracle_check": {"cells": int(c8.size), "max_ulp": ulp}, **card})
        del ser, out
        # TW48 from the daily tas, monthly output
        moff, yoff, ym, mdays = converters._months(ta)
        mtab = torch.from_numpy(converters._monthly_table("TW48", ta, ym, lat_u)).cuda()
        P = params("TW48", False, {"tas": (1.0, -273.15)})
        out = device.pet_monthly(ins(tas=tas), moff, yoff, mdays, mtab, idx_d, P)
        ms = timeit(lambda: device.pet_monthly(ins(tas=tas), moff, yoff, mdays, mtab, idx_d, P), a.steps)
        tsm = (sample(tas) * np.float32(1.0) + np.float32(-273.15)).astype(np.float32)
        ref = np.float32(PO.monthly_pet("TW48", ta.year, ta.month, ta.doy, "noleap", lat_u[idx[cols]], tas=tsm))
        got = out[:, cols].cpu().numpy()
        fin = np.isfinite(ref)
        ulp = float(np.max(np.abs(got[fin].view(np.int32).astype(np.int64) - ref[fin].view(np.int32).astype(np.int64))))
        report(f"pet TW48, {a.lat} x 1440 cells", ms, 4 * T * C + 4 * len(ym) * C,
               {"oracle_check": {"cells": int(cols.size), "max_ulp": ulp,
                                 "nan_match": bool(np.array_equal(np.isnan(got), np.isnan(ref)))}, **card})
        del out, tmin, tmax
    if want("etccdi") and a.only:   # day-of-year percentile indices: opt-in (--only etccdi)
        import subprocess
        from oracle import etccdi_oracle as EO
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True)
        card = {"gpu": torch.cuda.get_device_name(), "power_limit": q.stdout.strip() or "unknown",
                "frac_basis": "3.35 TB/s (H100 SXM data sheet)"}
        gt, gw = _lib.OPS[">"], _lib.RL_REDUCERS["sum"]

        def frac(nbytes, ms):
            return nbytes / (ms * 1e-3) / 3.35e12

        def rel(got, exp):
            got, exp = np.asarray(got, np.float64), np.asarray(exp, np.float64)
            with np.errstate(invalid="ignore", divide="ignore"):
                d = np.abs(got - exp) / np.maximum(np.abs(exp), 1e-30)
            return float(np.nanmax(np.where(np.isnan(got) & np.isnan(exp), 0.0, d)))

        # WSDI and tx90p on the full (10950, 721, 1440) grid, one lat tile at a time (30-year tx90 table per tile)
        del tas, pr
        torch.cuda.empty_cache()
        rows = 120
        tot = {"wsdi": 0.0, "tx90p": 0.0}
        nbytes = {"wsdi": 0, "tx90p": 0}
        worst, checked = 0, 0
        for r0 in range(0, 721, rows):
            nr = min(rows, 721 - r0)
            Ct = nr * X
            x = device.synth(T, Ct, kind=1, seed=3, cell_offset=r0 * X, cells_per_lat=X, n_lat_global=721)
            tab = device.percentile_doy(x, doy, yidx, YEAR, T // YEAR, 5, [90.0], 1 / 3, 1 / 3)[0]
            out, _ = device.doy_runstat(x, poff, doy, tab, gt, gw, 6, True)
            tot["wsdi"] += timeit(lambda: device.doy_runstat(x, poff, doy, tab, gt, gw, 6, True), a.steps)
            tot["tx90p"] += timeit(lambda: device.doy_threshold_count(x, poff, doy, tab, gt), a.steps)
            for k in tot:
                nbytes[k] += 4 * T * Ct + 8 * YEAR * Ct + 4 * (len(poff) - 1) * Ct
            if r0 == 0 or r0 + rows >= 721:          # sampled cells of the first and the last tile
                cols = np.unique(np.r_[np.linspace(0, Ct - 1, 64).astype(int), np.arange(Ct - 16, Ct)])
                exp = EO.warm_spell_duration_index(x[:, cols].cpu().numpy(), tab[:, cols].cpu().numpy(), doy, poff)
                worst = max(worst, int(np.sum(out[:, cols].cpu().numpy() != exp)))
                checked += cols.size
            del x, tab, out
            torch.cuda.empty_cache()
        for k, name in (("wsdi", "warm_spell_duration_index window 6"), ("tx90p", "tx90p count")):
            report(f"{name}, 721 x 1440 cells (lat tiles of {rows})", tot[k], nbytes[k],
                   {"grid": [T, 721, X], "cells_per_s": 721 * X / (tot[k] * 1e-3), "frac_of_3_35_tbs": frac(nbytes[k], tot[k]),
                    "wsdi_over_tx90p": tot["wsdi"] / tot["tx90p"],
                    "oracle_check": {"cells": checked, "mismatches": worst}, **card})
        # the band of --lat rows: fraction_over_precip_thresh, one compound index, DTR
        tas = device.synth(T, C, kind=1, seed=3, cells_per_lat=X, n_lat_global=a.lat)
        pr = device.synth(T, C, kind=0, seed=2, cells_per_lat=X, n_lat_global=a.lat)
        cols = np.unique(np.r_[np.linspace(0, C - 1, 96).astype(int), np.arange(C - 32, C)])
        ptab = torch.clamp(device.percentile_doy(pr, doy, yidx, YEAR, T // YEAR, 5, [95.0], 1 / 3, 1 / 3)[0], min=1.0)
        s_thr, s_wet = device.period_sums_thr(pr, poff, gt, ptab, 1.0, doy_index=doy)
        ms = timeit(lambda: device.period_sums_thr(pr, poff, gt, ptab, 1.0, doy_index=doy), a.steps)
        got = (s_thr / s_wet)[:, cols].cpu().numpy()
        exp = EO.fraction_over_precip_thresh(pr[:, cols].cpu().numpy(), ptab[:, cols].cpu().numpy(), 1.0, poff, doy=doy)
        nb = 4 * T * C + 8 * YEAR * C + 8 * (len(poff) - 1) * C
        report(f"fraction_over_precip_thresh (R95pTOT), {a.lat} x 1440 cells", ms, nb,
               {"frac_of_3_35_tbs": frac(nb, ms), "oracle_check": {"cells": int(cols.size), "max_rel_diff": rel(got, exp)},
                **card})
        del s_thr, s_wet
        ttab = device.percentile_doy(tas, doy, yidx, YEAR, T // YEAR, 5, [75.0], 1 / 3, 1 / 3)[0]
        ptab75 = device.percentile_doy(pr, doy, yidx, YEAR, T // YEAR, 5, [75.0], 1 / 3, 1 / 3)[0]
        lt = _lib.OPS["<"]
        out = device.doy_count2(tas, pr, poff, doy, ttab, ptab75, lt, gt)
        ms = timeit(lambda: device.doy_count2(tas, pr, poff, doy, ttab, ptab75, lt, gt), a.steps)
        exp = EO.compound_days("cold_and_wet_days", tas[:, cols].cpu().numpy(), pr[:, cols].cpu().numpy(),
                               ttab[:, cols].cpu().numpy(), ptab75[:, cols].cpu().numpy(), doy, poff)
        nb = 8 * T * C + 16 * YEAR * C + 4 * (len(poff) - 1) * C
        report(f"cold_and_wet_days, {a.lat} x 1440 cells", ms, nb,
               {"frac_of_3_35_tbs": frac(nb, ms),
                "oracle_check": {"cells": int(cols.size),
                                 "mismatches": int(np.sum(out[:, cols].cpu().numpy() != exp))}, **card})
        del ttab, ptab75, ptab, out
        torch.cuda.empty_cache()
        tmax = tas + torch.rand_like(tas) * 12
        for variability in (False, True):
            out = device.period_range_stat(tas, tmax, poff, _lib.STATS["mean"], variability)
            ms = timeit(lambda: device.period_range_stat(tas, tmax, poff, _lib.STATS["mean"], variability), a.steps)
            lo_s, hi_s = tas[:, cols].cpu().numpy(), tmax[:, cols].cpu().numpy()
            exp = EO.daily_temperature_range_variability(lo_s, hi_s, poff) if variability else \
                EO.daily_temperature_range(lo_s, hi_s, poff)
            nb = 8 * T * C + 4 * (len(poff) - 1) * C
            report(f"daily_temperature_range{'_variability' if variability else ''}, {a.lat} x 1440 cells", ms, nb,
                   {"frac_of_3_35_tbs": frac(nb, ms),
                    "oracle_check": {"cells": int(cols.size), "max_rel_diff": rel(out[:, cols].cpu().numpy(), exp)},
                    **card})
        del tmax, out
    if want("rainseason") and a.only:   # rain season: opt-in (--only rainseason), on the --lat band
        import subprocess

        from oracle import rain_season_oracle as RO
        from xclim_b200 import TimeAxis
        from xclim_b200.indices import _rain_season_mask
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True)
        card = {"gpu": torch.cuda.get_device_name(), "power_limit": q.stdout.strip() or "unknown",
                "frac_basis": "3.35 TB/s (H100 SXM data sheet)"}
        del tas, pr
        torch.cuda.empty_cache()
        # daily pr in mm/d: a rainy season of 10-day regimes (4 in 5 wet, 3-15 mm a day; the others 0-2 mm) between
        # a per-cell, per-year onset (doy 120-180) and cessation (doy 250-300), rare showers outside it, so that
        # most cells find a start after 05-01 and an end in a 20-day dry spell after 09-01 under the defaults
        g = torch.Generator(device="cuda").manual_seed(17)
        x = torch.empty((T, C), dtype=torch.float32, device="cuda")
        d = torch.arange(YEAR, device="cuda")[:, None]
        for y in range(T // YEAR):
            on = torch.randint(120, 181, (1, C), device="cuda", generator=g)
            off = torch.randint(250, 301, (1, C), device="cuda", generator=g)
            wet = (torch.rand((YEAR // 10 + 1, C), device="cuda", generator=g) < 0.8).repeat_interleave(10, 0)[:YEAR]
            u = torch.rand((YEAR, C), device="cuda", generator=g)
            season = (d >= on) & (d < off)
            shower = torch.rand((YEAR, C), device="cuda", generator=g) < 0.02
            x[y * YEAR:(y + 1) * YEAR] = torch.where(season, torch.where(wet, 3 + 12 * u, 2 * u),
                                                     torch.where(shower, 5 * u, torch.zeros_like(u)))
            del on, off, wet, u, season, shower
        ta = TimeAxis.daily("1991-01-01", T, "noleap")
        p = RO.DEFAULTS
        mask = _rain_season_mask(ta, poff, p["date_min_start"], p["date_max_start"], p["date_min_end"],
                                 p["date_max_end"])
        s, e = device.rain_season(x, poff, mask, 1.0, p["thresh_wet_start"], p["window_wet_start"],
                                  p["window_not_dry_start"], p["thresh_dry_start"], p["window_dry_start"],
                                  0, p["thresh_dry_end"], p["window_dry_end"], 0)
        # the kernel alone: the mask and the period offsets stay on the device between launches
        lib = _lib.load()
        mask_d = torch.from_numpy(mask).cuda()
        poff_d = torch.from_numpy(poff).cuda()
        st = torch.empty((P, C), dtype=torch.int32, device="cuda")
        en = torch.empty_like(st)

        def launch():
            _lib.check(lib.xc_rain_season_f32(x.data_ptr(), T, C, C, poff_d.data_ptr(), P, mask_d.data_ptr(), 1.0,
                                              25.0, 3, 30, 1.0, 7, 0, 0.0, 20, 0, st.data_ptr(), en.data_ptr(), None))
        ms = timeit(launch, a.steps)
        cols = np.unique(np.r_[np.linspace(0, C - 1, 96).astype(int), np.arange(C - 32, C)])
        o = RO.rain_season(x[:, cols].cpu().numpy(), ta, "YS")
        got_s = s[:, cols].cpu().numpy().astype(np.float64)
        got_e = e[:, cols].cpu().numpy().astype(np.float64)
        mism = int(np.sum(~np.isclose(np.where(got_s < 0, np.nan, got_s), o["start_idx"], equal_nan=True, rtol=0))
                   + np.sum(~np.isclose(np.where(got_e < 0, np.nan, got_e), o["end_idx"], equal_nan=True, rtol=0)))
        nb = T * C * 4 + 3 * P * C * 8
        report(f"rain_season (defaults), {a.lat} x 1440 cells", ms, nb,
               {"frac_of_3_35_tbs": nb / (ms * 1e-3) / 3.35e12,
                "seasons_found": float((s >= 0).float().mean()), "ends_found": float((e >= 0).float().mean()),
                "oracle_check": {"cells": int(cols.size), "mismatches": mism}, **card})
        del x, s, e, st, en
        torch.cuda.empty_cache()
    if want("chill") and a.only:   # chill portions and units: opt-in (--only chill), fused from daily tasmin/tasmax
        import subprocess

        from oracle import chill_oracle as CO
        from xclim_b200 import TimeAxis, converters
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True)
        card = {"gpu": torch.cuda.get_device_name(), "power_limit": q.stdout.strip() or "unknown"}
        del tas, pr
        torch.cuda.empty_cache()
        # daily tasmin / tasmax in degC over the band's latitudes (-89.75 .. -45.25 for 180 rows of a 0.25 grid):
        # a seasonal cycle of the cell's hemisphere plus noise, tasmax 2-14 degC above tasmin
        g = torch.Generator(device="cuda").manual_seed(23)
        ta = TimeAxis.daily("1991-01-01", T, "noleap")
        lats = -89.875 + 0.25 * np.arange(a.lat)
        season = torch.from_numpy(np.cos(2 * np.pi * (ta.doy - 15) / 365.0).astype(np.float32)).cuda()[:, None]
        lo = 2.0 + 8.0 * season + 4.0 * torch.randn((T, C), device="cuda", generator=g)
        hi = lo + 2.0 + 12.0 * torch.rand((T, C), device="cuda", generator=g)
        idx_np = np.repeat(np.arange(a.lat, dtype=np.int32), X)
        w = torch.from_numpy(converters.hourly_weights(ta, lats)).cuda()
        idx = torch.from_numpy(idx_np).cuda()
        poff_j = ta.period_offsets("YS-JUL")
        mask = ta.select_mask(date_bounds=("09-01", "03-30"))
        Pj = poff_j.size - 1
        lib = _lib.load()
        poff_d = torch.from_numpy(poff_j).cuda()
        mask_d = torch.from_numpy(mask.astype(np.uint8)).cuda()
        cp = torch.empty((Pj, C), dtype=torch.float64, device="cuda")
        cu = torch.empty((P, C), dtype=torch.float64, device="cuda")
        poff_y = torch.from_numpy(poff).cuda()

        def launch_cp():
            _lib.check(lib.xc_chill_daily_f32(lo.data_ptr(), hi.data_ptr(), T, C, C, w.data_ptr(), a.lat,
                                              idx.data_ptr(), poff_d.data_ptr(), Pj, mask_d.data_ptr(), 1.0, 273.15,
                                              1.0, 0.0, _lib.CHILL_PORTIONS, cp.data_ptr(), None, None, None))

        def launch_cu():
            _lib.check(lib.xc_chill_daily_f32(lo.data_ptr(), hi.data_ptr(), T, C, C, w.data_ptr(), a.lat,
                                              idx.data_ptr(), poff_y.data_ptr(), P, None, 1.0, 273.15, 1.0, 0.0,
                                              _lib.CHILL_UNITS, None, cu.data_ptr(), None, None))
        ms_cp = timeit(launch_cp, a.steps)
        ms_cu = timeit(launch_cu, a.steps)
        cols = np.unique(np.r_[np.linspace(0, C - 1, 6).astype(int), np.arange(C - 2, C)])
        lo_s, hi_s = lo[:, cols].cpu().numpy(), hi[:, cols].cpu().numpy()
        dl = converters.day_lengths(converters.day_angle(ta.year, ta.doy, "noleap")[:, None], lats[idx_np[cols]][None])
        hr = CO.hourly_temperature(lo_s, hi_s, dl)
        ocp, _, _ = CO.chill(hr, poff_j, mask, (1.0, 273.15), (1.0, 0.0))
        _, ocu, _ = CO.chill(hr, poff, None, (1.0, 273.15), (1.0, 0.0))
        got_cp, got_cu = cp[:, cols].cpu().numpy(), cu[:, cols].cpu().numpy()
        sel_hours = int(mask.sum()) * 24
        nb = 2 * T * C * 4 + Pj * C * 8
        report(f"chill_portions (fused, 09-01..03-30, YS-JUL), {a.lat} x 1440 cells", ms_cp, nb,
               {"selected_hours_per_cell": sel_hours, "fp64_exp_per_s": 4 * sel_hours * C / (ms_cp * 1e-3),
                "oracle_check": {"cells": int(cols.size),
                                 "max_rel_err": float(np.nanmax(np.abs(got_cp - ocp) / np.maximum(np.abs(ocp), 1e-300)))},
                **card})
        report(f"chill_units (fused, YS), {a.lat} x 1440 cells", ms_cu, 2 * T * C * 4 + P * C * 8,
               {"oracle_check": {"cells": int(cols.size), "mismatches": int(np.sum(got_cu != ocu))}, **card})
        del lo, hi, w, cp, cu
        torch.cuda.empty_cache()
    if want("bootspell") and a.only:   # bootstrapped WSDI: opt-in (--only bootspell), on the --lat band
        import subprocess

        from torch.profiler import ProfilerActivity, profile
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import fake_bootstrap   # the oracle-backed restatement of xc_bootstrap_doy_index_f32 (CPU)
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True)
        card = {"gpu": torch.cuda.get_device_name(), "power_limit": q.stdout.strip() or "unknown"}
        # warm_spell_duration_index(window=6, bootstrap=True) at per 90 over a 15-year base starting the series:
        # the bootstrapped periods of the base years, next to tx90p(bootstrap=True)'s count on the same input
        NB = 15
        sp = np.repeat(np.arange(NB), YEAR).astype(np.int32)
        P = T // YEAR
        gt = _lib.OPS[">"]

        def spell():
            return device.bootstrap_doy_index(tas, 0, NB, YEAR, sp, P, 5, 90.0, 1 / 3, 1 / 3, gt, "spell", 6)[0]

        def count():
            return device.bootstrap_doy_count(tas, 0, NB, YEAR, sp, P, 5, 90.0, 1 / 3, 1 / 3, gt)
        ms_spell = timeit(spell, a.steps)
        ms_count = timeit(count, a.steps)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            got = spell()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            for k in ("bootstrap5_kernel", "bootstrap_kernel", "bootstrap_reduce_kernel"):
                if k in e.key:
                    kern[k] = kern.get(k, 0.0) + e.device_time_total / 1000.0
        cols = np.unique(np.r_[np.linspace(0, C - 1, 2).astype(int), C - 1])
        xs = torch.from_numpy(tas[:NB * YEAR, cols].cpu().numpy())
        exp, _ = fake_bootstrap.bootstrap_doy_index(xs, 0, NB, YEAR, sp, P, 5, 90.0, 1 / 3, 1 / 3, gt, "spell", 6)
        ok = bool(np.array_equal(got[:NB, cols].cpu().numpy(), exp[:NB].numpy()))
        report(f"warm_spell_duration_index(window=6, bootstrap=True), 15-year base, {a.lat} x 1440 cells", ms_spell,
               NB * YEAR * C * 4 + NB * C * 8,
               {"ms_bootstrap_doy_count_same_input": ms_count, "ratio_to_count": ms_spell / ms_count,
                "kernel_ms": kern, "oracle_check": {"cells": int(cols.size), "bit_exact": ok}, **card})
    if want("fwi") and a.only:      # the fire-weather kernel: opt-in (--only fwi), never part of a default run
        import time

        from xclim_b200 import fire
        # degC / mm/d / % / km/h series from the generators above; humidity and wind from hashed noise
        tas_c = tas - 273.15
        hurs = device.synth(T, C, kind=1, seed=11, cells_per_lat=X, n_lat_global=a.lat)
        hurs = ((hurs - hurs.mean()) * 4.0 + 55.0).clamp_(5.0, 100.0)
        ws = (device.synth(T, C, kind=1, seed=12, cells_per_lat=X, n_lat_global=a.lat) - 270.0).abs_().mul_(0.5)
        month = (np.minimum((np.arange(T) % YEAR) // 30.42, 11) + 1).astype(np.int8)
        lat = np.repeat(np.linspace(-60, 75, a.lat), X)
        p = {k: (v if not isinstance(v, tuple) else v[0]) for k, v in fire.default_params.items()}
        for label, outs, kw in (
                ("fwi always-on, 6 outputs", ["DC", "DMC", "FFMC", "ISI", "BUI", "FWI"], {}),
                ("fwi WF93 season, 6 outputs + mask", ["DC", "DMC", "FFMC", "ISI", "BUI", "FWI", "season_mask"],
                 {"season_method": "WF93"}),
                ("fwi drought code only", ["DC"], {})):
            P = device.fwi_params(kw.get("season_method"), False, None, True, **p)
            need = [tas_c, pr] + ([hurs, ws] if len(outs) > 1 else [None, None])
            run = lambda: device.fire_weather(need[0], need[1], need[2], need[3], None, month, lat, None, None, None,  # noqa: E731
                                              None, None, outs, P)
            ms = timeit(run, a.steps)
            n_in = sum(x is not None for x in need)
            n_out = sum(o != "season_mask" for o in outs)
            extra = {"bound": "FP64 pipe (about twenty float64 transcendentals per element)"}
            if a.cpu:
                from oracle import fire_oracle as FO
                Sf = min(S, 256)
                hh = [None if x is None else x[:, :Sf].cpu().numpy() for x in need]
                t0 = time.perf_counter()
                FO.fire_weather_calc(hh[0], hh[1], hh[2], hh[3], None, month, lat[:Sf], None,
                                     *(np.full(Sf, np.nan, np.float32),) * 3, np.zeros(Sf, np.float32),
                                     outputs=FO.complete_indexes([o for o in outs if o != "season_mask"])
                                     + (["season_mask"] if "season_mask" in outs else []), **kw)
                dt = time.perf_counter() - t0
                extra["cpu_port"] = {"cells_per_s": Sf / dt, "cores": 1, "kind": "port", "sample": f"({T}, {Sf}) cells, {dt:.1f} s"}
            report(label, ms, (n_in + n_out) * T * C * 4 + (T * C if "season_mask" in outs else 0), extra)
    if want("ens") and a.only:      # ensemble statistics: opt-in (--only ens), on their own full-grid inputs
        import subprocess

        from oracle import ensemble_oracle as EO
        del tas, pr
        torch.cuda.empty_cache()
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True)
        card = {"gpu": torch.cuda.get_device_name(), "power_limit": q.stdout.strip() or "unknown"}
        g = torch.Generator(device="cuda").manual_seed(5)
        years, grid = 150, 721 * 1440
        per = [10, 50, 90]
        # an annual indicator of R members over 150 years on the full grid, then R = 100 on a band that fits
        for R, rows in ((30, 721), (100, 180)):
            N = years * rows * 1440
            x = torch.randn((R, N), generator=g, device="cuda", dtype=torch.float32).mul_(3.0).add_(285.0)
            out = device.ens_percentiles(x, per, 1.0, 1.0, 1)
            ms = timeit(lambda: device.ens_percentiles(x, per, 1.0, 1.0, 1), a.steps)
            cols = np.r_[np.arange(0, N, max(1, N // 509)), N - 1]
            got = out[:, cols].cpu().numpy()
            exp = EO.percentiles(x[:, cols].cpu().numpy(), per)
            report(f"ens_percentiles R={R} (10, 50, 90), {years} years x {rows} x 1440", ms, R * N * 4 + len(per) * N * 8,
                   {"columns": N, "path": "registers" if R <= 32 else "shared memory",
                    "oracle_check": {"cells": int(cols.size), "bit_equal": bool(np.array_equal(got, exp))}, **card})
            del x, out
            torch.cuda.empty_cache()
        R, Ty = 30, 30
        fut = torch.randn((R, Ty, grid), generator=g, device="cuda", dtype=torch.float32).add_(0.3)
        ref = torch.randn((R, Ty, grid), generator=g, device="cuda", dtype=torch.float32)
        code = _lib.ENS_TESTS["ttest"]
        frac, pv = device.ens_robustness(fut, ref, None, code, 0.05, True, True)
        ms = timeit(lambda: device.ens_robustness(fut, ref, None, code, 0.05, True, True), a.steps)
        cols = np.r_[np.arange(0, grid, grid // 127), grid - 1]
        exp, p, _ = EO.robustness(fut[:, :, cols].cpu().numpy(), ref[:, :, cols].cpu().numpy(), "ttest")
        fr = frac[:, cols].cpu().numpy()
        pk = pv[:, cols].cpu().numpy()
        pos = p > 0                                   # p = 0 (t = +-inf) has no relative difference
        check = {"cells": int(cols.size),
                 "fractions_equal": bool(all(np.array_equal(fr[k], exp[n]) for k, n in enumerate(EO.FRACTIONS))),
                 "pvals_zero_and_nan_equal": bool(np.array_equal(pk == 0, p == 0)
                                                  and np.array_equal(np.isnan(pk), np.isnan(p))),
                 "max_pval_rel_diff_f32": float(np.max(np.abs(pk[pos] - p[pos]) / p[pos])) if pos.any() else 0.0}
        report(f"ens_robustness ttest R={R}, {Ty} + {Ty} years x 721 x 1440", ms, 2 * R * Ty * grid * 4 + 7 * grid * 8
               + R * grid * 4, {"cells": grid, "oracle_check": check, **card})


if __name__ == "__main__":
    main()
