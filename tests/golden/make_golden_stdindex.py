"""Generate tests/golden/ref_stdindex.npz: the reference's own distribution fit on hand-picked samples.

Runs ``_fitfunc_1d``, ``_fit_start`` and ``get_dist`` of indices/stats.py where they lie (``_ref_extract``), with
scipy's distributions, and stores inputs and outputs only.  Usage:
``XCLIM_REFERENCE_ROOT=/path/to/xclim python tests/golden/make_golden_stdindex.py``.

Cases: every supported dist x method x zero inflation; sample lengths 0, 1, 2, 7, 8, 9, 30, 127, 128, 129, 300 (the
edges of numpy's pairwise summation); constant and tied samples; values at 1e-30 and 1e30, +-inf and NaN; negative
values with floc = 0 (APP drops them, ML raises).  Zero inflation is applied as the reference applies it before the
fit (stats.py:947, ``da.where(da != 0)``).
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import _ref_extract  # noqa: E402

CASES = [("gamma", "APP"), ("gamma", "ML"), ("fisk", "APP"), ("lognorm", "APP"), ("lognorm", "ML")]
NMAX = 300


def load_fit():
    import scipy.stats
    from typing import Any

    from scipy.stats import rv_continuous
    ns = {"np": np, "scipy": scipy, "rv_continuous": rv_continuous, "Any": Any, "warnings": warnings}
    return _ref_extract._extract("src/xclim/indices/stats.py", ["_fitfunc_1d", "_fit_start", "get_dist"], ns)


def samples():
    rng = np.random.default_rng(20261016)
    out = []
    for n in (0, 1, 2, 7, 8, 9, 30, 127, 128, 129, 300):
        v = rng.gamma(0.9, 25.0, n).astype(np.float32)
        v[rng.random(n) < 0.2] = 0.0
        out.append(("n%d" % n, v))
    out.append(("constant", np.full(12, 2.5, np.float32)))
    out.append(("tied", np.array([1, 1, 1, 2, 2, 3, 3, 3, 3], np.float32)))
    out.append(("tiny", np.array([1e-30, 3e-30, 2e-30, 5e-30, 1e-29], np.float32)))
    out.append(("huge", np.array([1e30, 3e30, 2e30, 5e30, 1e29, 7e30], np.float32)))
    out.append(("nonfinite", np.array([np.inf, 3.0, np.nan, 4.5, -np.inf, 0.0, 7.25, 1.5], np.float32)))
    out.append(("negatives", np.array([-2.0, 3.0, 1.0, -0.5, 4.0, 0.0, 6.0], np.float32)))
    out.append(("all_zero", np.zeros(10, np.float32)))
    return out


def main():
    ref = _ref_extract
    if not ref.available():
        raise SystemExit("set XCLIM_REFERENCE_ROOT to a checkout of the reference")
    f = load_fit()
    smp = samples()
    names, x, n = [], np.full((len(smp), NMAX), np.nan, np.float32), np.zeros(len(smp), np.int32)
    for i, (name, v) in enumerate(smp):
        names.append(name)
        x[i, :v.size] = v
        n[i] = v.size
    params = np.full((len(CASES), 2, len(smp), 3), np.nan)
    error = np.zeros((len(CASES), 2, len(smp)), np.int8)      # 0 ok, 1 ValueError, 2 other exception
    for ci, (dist, method) in enumerate(CASES):
        for zi in (0, 1):
            for i in range(len(smp)):
                v = x[i, :n[i]]
                if zi:
                    v = np.where(v != 0, v, np.float32(np.nan))
                with warnings.catch_warnings(), np.errstate(all="ignore"):
                    warnings.simplefilter("ignore")
                    try:
                        params[ci, zi, i] = f["_fitfunc_1d"](v, dist=f["get_dist"](dist), nparams=3, method=method,
                                                            floc=0.0)
                    except ValueError:
                        error[ci, zi, i] = 1
                    except Exception:  # noqa: BLE001 - recorded, not hidden
                        error[ci, zi, i] = 2
    np.savez_compressed(os.path.join(HERE, "ref_stdindex.npz"), x=x, n=n, names=np.array(names),
                        dists=np.array([c[0] for c in CASES]), methods=np.array([c[1] for c in CASES]),
                        params=params, error=error)


if __name__ == "__main__":
    main()
