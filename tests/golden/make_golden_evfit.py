"""Generate tests/golden/ref_evfit.npz: the reference's own maximum-likelihood fits on hand-picked samples.

Runs ``_fitfunc_1d``, ``_fit_start`` and ``get_dist`` of indices/stats.py where they lie (``_ref_extract``), with
scipy's distributions, and stores inputs and outputs only, with the scipy version that made them.  Usage:
``XCLIM_REFERENCE_ROOT=/path/to/xclim python tests/golden/make_golden_evfit.py``.

Cases: sample lengths 0, 1, 2, 3, 7, 8, 9, 30, 127, 128, 129, 300 (the edges of numpy's pairwise summation);
ties and constant samples; NaN and +-inf mixed in; values near 1e-30 and 1e30; the reference test's GEV
fixture (tests/test_stats.py ``genextreme``); heavy-tailed (c = -0.4) and bounded (c = 0.3) GEV samples.
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import _ref_extract  # noqa: E402

DISTS = ["norm", "gumbel_r", "genextreme"]
NMAX = 300
#: the reference test's GEV fixture and its known answer (tests/test_stats.py: genextreme, test_genextreme_fit)
GEV_FIXTURE = [279, 302, 450, 272, 401, 222, 311, 327, 294, 299, 348, 286, 492, 296, 227, 437, 340, 376, 444, 177]


def load_fit():
    import scipy.stats
    from typing import Any

    from scipy.stats import rv_continuous
    ns = {"np": np, "scipy": scipy, "rv_continuous": rv_continuous, "Any": Any, "warnings": warnings}
    return _ref_extract._extract("src/xclim/indices/stats.py", ["_fitfunc_1d", "_fit_start", "get_dist"], ns)


def samples():
    import scipy.stats as st
    rng = np.random.default_rng(20261017)
    out = []
    for n in (0, 1, 2, 3, 7, 8, 9, 30, 127, 128, 129, 300):
        out.append(("n%d" % n, st.genextreme.rvs(-0.1, loc=30, scale=8, size=n, random_state=rng)
                    .astype(np.float32)))
    out.append(("constant", np.full(12, 2.5, np.float32)))
    out.append(("constant_inexact", np.full(7, 0.1, np.float32)))
    out.append(("tied", np.array([1, 1, 1, 2, 2, 3, 3, 3, 3, 5, 5, 8], np.float32)))
    out.append(("nonfinite", np.array([np.inf, 31.0, np.nan, 44.5, -np.inf, 27.0, 37.25, 51.5, np.nan, 29.0,
                                       35.5, 40.0], np.float32)))
    out.append(("tiny", (rng.gumbel(3.0, 1.0, 40) * 1e-30).astype(np.float32)))
    out.append(("huge", (rng.gumbel(3.0, 1.0, 40) * 1e30).astype(np.float32)))
    out.append(("ref_fixture", np.array(GEV_FIXTURE, np.float32)))
    for n in (30, 150):
        out.append(("heavy%d" % n, st.genextreme.rvs(-0.4, loc=30, scale=8, size=n, random_state=rng)
                    .astype(np.float32)))
        out.append(("bounded%d" % n, st.genextreme.rvs(0.3, loc=30, scale=8, size=n, random_state=rng)
                    .astype(np.float32)))
    return out


def main():
    import scipy
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
    params = np.full((len(DISTS), len(smp), 3), np.nan)
    error = np.zeros((len(DISTS), len(smp)), np.int8)       # 0 ok, 1 ValueError, 2 other exception
    for di, dist in enumerate(DISTS):
        for i in range(len(smp)):
            v = x[i, :n[i]]
            with warnings.catch_warnings(), np.errstate(all="ignore"):
                warnings.simplefilter("ignore")
                try:
                    p = f["_fitfunc_1d"](v, dist=f["get_dist"](dist), nparams=3 if dist == "genextreme" else 2,
                                         method="ML")
                    params[di, i, :p.size] = p
                except ValueError:
                    error[di, i] = 1
                except Exception:  # noqa: BLE001 - recorded, not hidden
                    error[di, i] = 2
    np.savez_compressed(os.path.join(HERE, "ref_evfit.npz"), x=x, n=n, names=np.array(names),
                        dists=np.array(DISTS), params=params, error=error, scipy_version=scipy.__version__)


if __name__ == "__main__":
    main()
