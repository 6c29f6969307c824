"""The standardized-index fit against the reference's own code (tests/golden/ref_stdindex.npz, made by
make_golden_stdindex.py from indices/stats.py `_fitfunc_1d` / `_fit_start` / `get_dist` with scipy).

* oracle/stdindex_oracle.py with ``numpy_logs=True`` (numpy's float32 log / exp, as the reference) matches the
  stored parameters bit for bit and raises where the reference raised;
* the host build of the kernels' code (float64 logs rounded once to float32) agrees within the conditioning of
  the moment expressions: a float32 log differs from numpy's by at most an ulp, and A = log(mean) - mean(log)
  (gamma), the log-standard deviation (lognorm) or s (gamma ML) turn that ulp into a relative error of the shape
  of about ulp(|log m|) / |A|."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import stdindex_host_build as H  # noqa: E402
from oracle import stdindex_oracle as O  # noqa: E402

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")
G = np.load(os.path.join(HERE, "golden", "ref_stdindex.npz"))
CASES = list(zip(G["dists"], G["methods"]))


def _sample(i, zi):
    v = G["x"][i, :G["n"][i]]
    return np.where(v != 0, v, np.float32(np.nan)) if zi else v


@pytest.mark.parametrize("ci", range(len(CASES)))
@pytest.mark.parametrize("zi", [0, 1])
def test_oracle_numpy_logs_matches_reference_bit_for_bit(ci, zi):
    dist, method = (str(s) for s in CASES[ci])
    for i, name in enumerate(G["names"]):
        err = int(G["error"][ci, zi, i])
        try:
            p = O.fit_sample(_sample(i, zi), dist, method, 0.0, numpy_logs=True)
        except NotImplementedError:
            # lognorm ML on a sample of zero spread: the reference hands it to scipy's generic optimiser
            assert (dist, method) == ("lognorm", "ML") and err == 0, name
            continue
        except ValueError:
            assert err == 1, name
            continue
        assert err == 0, name
        np.testing.assert_array_equal(p, G["params"][ci, zi, i], err_msg=str(name))


def _shape_tol(dist, method, v, p_ref):
    """Relative tolerance of the shape between the two log rules (see the module docstring)."""
    x = v[np.isfinite(v) & (v > 0)].astype(np.float64)
    lx = np.log(x)
    ulp_log = 2.0 ** -23 * (np.abs(np.log(x.mean())) + np.abs(lx).mean() + 1.0)
    if dist == "gamma":
        A = np.log(x.mean()) - lx.mean()
        return 4 * ulp_log / max(abs(A), 1e-300) + 1e-6
    if dist == "lognorm":
        return 4 * ulp_log / max(lx.std(), 1e-300) ** 2 + 1e-6
    return 1e-6


@pytest.mark.parametrize("ci", range(len(CASES)))
@pytest.mark.parametrize("zi", [0, 1])
def test_kernel_log_rule_against_reference(ci, zi):
    dist, method = (str(s) for s in CASES[ci])
    S = len(G["names"])
    y = np.full((300, S), np.nan, np.float32)
    for i in range(S):
        y[:G["n"][i], i] = G["x"][i, :G["n"][i]]
    gos = np.zeros(300, int)
    for i, name in enumerate(G["names"]):
        err = int(G["error"][ci, zi, i])
        p, _, _, st = H.fit(y[:, i:i + 1], gos, 1, dist, method, bool(zi), 0.0)
        ref = G["params"][ci, zi, i]
        if err:
            assert st & (1 | 2 | 4), name        # the call raises ValueError, as the reference does
            continue
        if st & 8:
            assert (dist, method) == ("lognorm", "ML"), name
            continue
        if st:
            # the reference's own (numpy) logs found a root where the kernel's rounding gives s <= 0: only on a
            # constant sample, where s is a difference of two equal logs
            assert (dist, method, str(name)) == ("gamma", "ML", "constant"), name
            continue
        got = p[0, :, 0]
        np.testing.assert_array_equal(np.isnan(got), np.isnan(ref), err_msg=str(name))
        if np.isnan(ref).all():
            continue
        assert got[1] == ref[1]
        v = _sample(i, zi)
        if not np.isfinite(ref[0]):
            assert got[0] == ref[0] and got[2] == ref[2], name
            continue
        tol = _shape_tol(dist, method, v, ref)
        assert abs(got[0] - ref[0]) <= tol * abs(ref[0]), (name, got, ref, tol)
        assert abs(got[2] - ref[2]) <= (tol + 2.0 ** -22) * abs(ref[2]), (name, got, ref, tol)
