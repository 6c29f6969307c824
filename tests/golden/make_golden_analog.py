"""Generate tests/golden/ref_analog.npz: the reference's own dissimilarity metrics on hand-picked samples.

Runs ``metric`` (with ``_metric_overhead``), ``standardize`` and the metric functions of analog.py where they lie
(``_ref_extract``), with scipy, and stores inputs and outputs only, with the scipy version that made them.  Usage:
``XCLIM_REFERENCE_ROOT=/path/to/xclim python tests/golden/make_golden_analog.py``.

Cases: sample sizes n, m in {5, 6, 30, 31, 64} (n != m) with d in {1, 2, 3, 10}, in float32 and float64;
integer-valued samples (ties, duplicates, zero distances); a constant indicator in either sample; +-inf and NaN in
either sample (recording which raise and with what message); values near 1e-30 and 1e30; the reference tests'
``matlab_sample``.
"""
from __future__ import annotations

import functools
import os
import sys
import warnings
from collections.abc import Callable, Sequence
from typing import Any

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import _ref_extract  # noqa: E402

#: (column name, metric, kwargs)
COLUMNS = [("seuclidean", "seuclidean", {}), ("nearest_neighbor", "nearest_neighbor", {}),
           ("zech_aslan", "zech_aslan", {}), ("szekely_rizzo", "szekely_rizzo", {}),
           ("szekely_rizzo_raw", "szekely_rizzo", {"standardize": False}),
           ("kolmogorov_smirnov", "kolmogorov_smirnov", {}), ("kldiv", "kldiv", {}),
           ("kldiv_k3", "kldiv", {"k": 3}), ("mahalanobis", "mahalanobis", {})]


def load_metrics():
    from scipy import spatial
    from scipy.spatial import cKDTree
    ns = {"np": np, "spatial": spatial, "KDTree": cKDTree, "wraps": functools.wraps, "Callable": Callable,
          "Sequence": Sequence, "Any": Any}
    names = ["metrics", "standardize", "metric", "seuclidean", "nearest_neighbor", "zech_aslan", "szekely_rizzo",
             "friedman_rafsky", "kolmogorov_smirnov", "kldiv", "mahalanobis"]
    return _ref_extract._extract("src/xclim/analog.py", names, ns)["metrics"]


def matlab_sample(n=30):
    """tests/test_analog.py ``matlab_sample``."""
    z = 1.0 * (np.arange(n) + 1) / n - 0.5
    return np.vstack([z * 2 + 30, z * 3 + 40, z]).T, np.vstack([z * 2.2 + 31, z[::-1] * 2.8 + 38, z * 1.1]).T


def samples():
    rng = np.random.default_rng(20261017)
    out = []
    pairs = [(5, 6), (6, 5), (30, 31), (31, 64), (64, 30)]
    for n, m in pairs:
        for d in (1, 2, 3, 10):
            x = rng.normal(10.0, 2.0, (n, d))
            y = rng.normal(10.5, 2.5, (m, d)) + rng.normal(0, 0.5, d)
            for dt in (np.float32, np.float64):
                out.append((f"normal_n{n}_m{m}_d{d}_{np.dtype(dt).name}", x.astype(dt), y.astype(dt)))
    for dt in (np.float32, np.float64):
        nm = np.dtype(dt).name
        out.append((f"integer_{nm}", rng.integers(0, 4, (30, 3)).astype(dt), rng.integers(0, 5, (31, 3)).astype(dt)))
        out.append((f"integer_d1_{nm}", rng.integers(0, 3, (31, 1)).astype(dt), rng.integers(0, 3, (6, 1)).astype(dt)))
        x = rng.normal(5, 1, (30, 3)).astype(dt)
        y = rng.normal(5, 1, (31, 3)).astype(dt)
        x[7], y[3] = x[2], x[2]                                  # duplicates within and across samples
        out.append((f"duplicates_{nm}", x, y))
        xc = x.copy()
        xc[:, 1] = 5
        out.append((f"const_target_{nm}", xc, y))
        yc = y.copy()
        yc[:, 0] = 5
        out.append((f"const_cand_{nm}", x, yc))
        for where in ("target", "cand"):
            for val, tag in ((np.inf, "posinf"), (-np.inf, "neginf"), (np.nan, "nan")):
                a, b = x.copy(), y.copy()
                (a if where == "target" else b)[4, 1] = val
                out.append((f"{tag}_{where}_{nm}", a, b))
        a = x[:4].copy()
        a[1, 0] = np.inf
        out.append((f"posinf_small_target_{nm}", a, y))          # kldiv: n < 5 answers NaN before the inf check
    for scale in (1e-30, 1e30):
        out.append((f"scale_{scale:g}_float64", rng.normal(3, 1, (30, 3)) * scale, rng.normal(3.3, 1.2, (31, 3)) * scale))
    x, y = matlab_sample()
    out.append(("matlab_sample", x, y))
    return out


def main():
    import scipy
    if not _ref_extract.available():
        raise SystemExit("set XCLIM_REFERENCE_ROOT to a checkout of the reference")
    metrics = load_metrics()
    smp = samples()
    store = {}
    values = np.full((len(smp), len(COLUMNS)), np.nan)
    errors = np.full((len(smp), len(COLUMNS)), "", dtype=object)
    for i, (name, x, y) in enumerate(smp):
        store[f"x_{i}"], store[f"y_{i}"] = x, y
        for j, (_, meth, kw) in enumerate(COLUMNS):
            with warnings.catch_warnings(), np.errstate(all="ignore"):
                warnings.simplefilter("ignore")
                try:
                    values[i, j] = metrics[meth](x, y, **kw)
                except Exception as e:  # noqa: BLE001 - recorded, not hidden
                    errors[i, j] = f"{type(e).__name__}: {e}"
    np.savez_compressed(os.path.join(HERE, "ref_analog.npz"), names=np.array([s[0] for s in smp]),
                        columns=np.array([c[0] for c in COLUMNS]), values=values, errors=errors.astype(str),
                        metrics=np.array(list(metrics)), scipy_version=scipy.__version__, **store)


if __name__ == "__main__":
    main()
