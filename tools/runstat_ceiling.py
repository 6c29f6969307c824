"""HBM read ceiling of the headline run statistic (maximum_consecutive_dry_days + the MissingAny valid count on
(10950, 721, 1440) float32, yearly periods), against read-only reductions of the same buffer.  One GPU.

    python tools/runstat_ceiling.py [--reps 3] [--calls 10] [--lat 721]

Prints the card, its power limit and SM clocks, then for each variant, timed with CUDA events in rounds that
alternate the variants (one warm-up call each per round), the median ms per call, the rate in TB/s of the bytes the
call must move (the input once; the run statistic also writes its two (30, C) outputs) and the spread over rounds:
  runstat         the dispatch as it stands (the bulk-copy kernel on this shape)
  runstat_v1      the per-lane period_runstat_kernel (XCLIM_B200_RUNSTAT_V1=1)
  sum_time        torch.sum(pr, dim=0): one read of every element, reduced over time
  sum_flat        torch.sum(pr): one read of every element, reduced to a scalar
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

T, X, YEAR = 10950, 1440, 365


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--lat", type=int, default=721)
    a = ap.parse_args()

    import torch

    from xclim_b200 import _lib, device

    C = a.lat * X
    P = T // YEAR
    poff = np.arange(P + 1, dtype=np.int32) * YEAR
    pr = device.synth(T, C, kind=0, seed=2, cells_per_lat=X, n_lat_global=a.lat)
    op, red = _lib.OPS["<"], _lib.RL_REDUCERS["max"]
    read = T * C * 4
    io = read + 2 * P * C * 4

    def runstat():
        return device.period_runstat(pr, poff, op, 1.0, red, 1, True, want_valid=True)

    def with_v1(fn):
        def g():
            os.environ["XCLIM_B200_RUNSTAT_V1"] = "1"
            try:
                return fn()
            finally:
                del os.environ["XCLIM_B200_RUNSTAT_V1"]
        return g

    os.environ.pop("XCLIM_B200_RUNSTAT_V1", None)
    variants = {"runstat": (runstat, io), "runstat_v1": (with_v1(runstat), io),
                "sum_time": (lambda: torch.sum(pr, dim=0), read), "sum_flat": (lambda: torch.sum(pr), read)}
    new, old = runstat(), with_v1(runstat)()
    same = bool(torch.equal(new[0].view(torch.int32), old[0].view(torch.int32)) and torch.equal(new[1], old[1]))
    del new, old
    print(f"card: {card()}")
    print(f"input (T, C) = ({T}, {C}) float32, {read / 1e9:.2f} GB; runstat moves {io / 1e9:.2f} GB; "
          f"bulk and per-lane outputs identical: {same}")
    ms = {k: [] for k in variants}
    for _ in range(a.reps):
        for name, (fn, _) in variants.items():
            fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.calls):
                fn()
            e1.record()
            e1.synchronize()
            ms[name].append(e0.elapsed_time(e1) / a.calls)
    res = {}
    for name, (_, nbytes) in variants.items():
        v = np.array(ms[name])
        med = float(np.median(v))
        res[name] = {"ms": med, "tb_s": nbytes / (med * 1e-3) / 1e12, "spread_ms": float(v.max() - v.min()),
                     "rounds_ms": [round(float(t), 3) for t in v]}
        print(f"{name:11s} {med:8.3f} ms  {res[name]['tb_s']:.3f} TB/s  spread {res[name]['spread_ms']:.3f} ms  "
              f"rounds {res[name]['rounds_ms']}")
    print(f"card after: {card()}")
    print(json.dumps({"card": card(), "identical": same, "results": res}))


if __name__ == "__main__":
    main()
