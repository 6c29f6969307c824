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


if __name__ == "__main__":
    main()
