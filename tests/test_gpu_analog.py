"""Spatial analogues on the GPU: the kernel against the host build of the same device code
(tests/csrc/analog_host.cpp) on grids around whole CTAs, strided views, several targets and hostile cells, and
spatial_analogs end to end from tg_mean / frost_days indicators against the oracle."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import analog_host_build as H  # noqa: E402
from oracle import analog_oracle as O  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]

#: method -> (kernel params to run, bit for bit?)
METHODS = {"seuclidean": ([0.0], False), "nearest_neighbor": ([0.0], True), "zech_aslan": ([1e-12, 1e-3], False),
           "szekely_rizzo": ([1.0, 0.0], False), "kolmogorov_smirnov": ([0.0], True), "kldiv": ([1.0, 3.0], False),
           "mahalanobis": ([0.0], False)}


def _consts(t, method):
    if method not in ("seuclidean", "mahalanobis"):
        return None
    if method == "mahalanobis" and t.shape[2] == 1:     # one indicator: the reference needs a user VI
        return np.stack([1.0 / x.var(ddof=1, keepdims=True).ravel() for x in t.astype(np.float64)])
    return np.stack([np.asarray(O.target_consts(x, method)).ravel() for x in t.astype(np.float64)])


def _hostile(y, rng):
    """Mix NaN, +-inf, constant and integer-valued (tied) cells into a (C, m, d) sample."""
    C = y.shape[0]
    cells = rng.choice(C, size=min(C, 6), replace=False)
    kinds = ["nan", "posinf", "neginf", "const", "int", "dup"]
    for c, kind in zip(cells, kinds):
        if kind == "nan":
            y[c, 2, 0] = np.nan
        elif kind == "posinf":
            y[c, 1, -1] = np.inf
        elif kind == "neginf":
            y[c, 0, 0] = -np.inf
        elif kind == "const":
            y[c, :, 0] = 3.0
        elif kind == "int":
            y[c] = np.round(y[c])
        else:
            y[c, 1] = y[c, 0]
    return y


def _run(t, y, method, param, ldc_pad=0):
    """The kernel on (K, n, d) targets and (C, m, d) candidates laid out (m, d, C) in a buffer of row ldc."""
    import torch
    from xclim_b200 import _lib, device
    K, n, d = t.shape
    C, m, _ = y.shape
    buf = torch.full((m, d, C + ldc_pad), 7.0, dtype=torch.float32, device="cuda")
    buf[:, :, :C] = torch.from_numpy(np.ascontiguousarray(np.moveaxis(y, 0, -1))).cuda()
    cand = buf[:, :, :C]
    cst = _consts(t, method)
    cst = None if cst is None else torch.from_numpy(cst).cuda()
    out, status = device.analog(torch.from_numpy(t).cuda(), cand, _lib.AN_METHODS[method], param, cst)
    return out.cpu().numpy(), status


def _compare(got, want, exact):
    special = ~np.isfinite(want)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    np.testing.assert_array_equal(got[special & ~np.isnan(want)], want[special & ~np.isnan(want)])
    if exact:
        np.testing.assert_array_equal(got, want)
    else:
        np.testing.assert_allclose(got[~special], want[~special], rtol=1e-13, atol=1e-13)


@pytest.mark.parametrize("method", list(METHODS))
@pytest.mark.parametrize("C, K, n, m, d, pad", [(1, 1, 30, 30, 3, 0), (31, 3, 30, 31, 3, 0), (32, 1, 6, 5, 1, 5),
                                                (33, 3, 31, 64, 2, 0), (4100, 1, 30, 30, 3, 3),
                                                (65, 1, 64, 30, 10, 0)])
def test_kernel_matches_host_build(method, C, K, n, m, d, pad):
    rng = np.random.default_rng(C * 7 + K + d)
    t = rng.normal(10, 2, (K, n, d)).astype(np.float32)
    y = (rng.normal(10.5, 2.5, (C, m, d)) + rng.normal(0, 1, (C, 1, d))).astype(np.float32)
    if C > 1:
        y = _hostile(y, rng)
    if K > 1:
        t[1] = np.round(t[1])                   # an integer-valued (tied) target
    params, exact = METHODS[method]
    for param in params:
        got, st = _run(t, y, method, param, pad)
        want, wst = H.analog(t, y, method, param, _consts(t, method))
        assert st == wst, (method, param)
        _compare(got, want, exact)


def test_every_method_on_integer_samples_and_ldc_view():
    """Integer-valued indicators: ties and zero distances everywhere (kldiv +-inf / NaN, nearest-neighbour ties)."""
    rng = np.random.default_rng(9)
    t = rng.integers(0, 4, (1, 30, 3)).astype(np.float32)
    y = rng.integers(0, 5, (300, 31, 3)).astype(np.float32)
    for method, (params, exact) in METHODS.items():
        for param in params:
            got, st = _run(t, y, method, param, ldc_pad=17)
            want, wst = H.analog(t, y, method, param, _consts(t, method))
            assert st == wst
            _compare(got, want, exact or method == "kldiv")


@pytest.mark.parametrize("calendar", ["noleap", "standard"])
def test_spatial_analogs_end_to_end(calendar):
    from xclim_b200 import analog, indices
    from xclim_b200.field import Field
    from xclim_b200.timeaxis import TimeAxis
    rng = np.random.default_rng(12)
    years, nx, ny = 30, 5, 7
    T = sum(366 if (calendar == "standard" and (y % 4 == 0 and (y % 100 != 0 or y % 400 == 0))) else 365
            for y in range(1981, 1981 + years))
    ta = TimeAxis.daily("1981-01-01", T, calendar)
    doy = np.arange(T) % 365
    base = 280 + 12 * np.sin(2 * np.pi * (doy - 100) / 365)[:, None, None]
    tas = (base + rng.normal(0, 4, (T, nx, ny)) + np.linspace(-8, 8, nx)[None, :, None]).astype(np.float32)
    tasmin = (tas - 5 + rng.normal(0, 1, tas.shape)).astype(np.float32)
    tg = indices.tg_mean(Field(tas, ("time", "x", "y"), ta, {}, {"units": "K"}))
    fd = indices.frost_days(Field(tasmin, ("time", "x", "y"), ta, {}, {"units": "K"}))
    cand = {"tg_mean": tg, "frost_days": fd}
    tv = {k: np.asarray(v.values)[:20, 2, 3] for k, v in cand.items()}
    target = {k: Field(v, ("time",), None, {}, {}, k) for k, v in tv.items()}
    cv = np.stack([np.asarray(v.values) for v in cand.values()], -1).astype(np.float64)     # (time, x, y, d)
    tx = np.stack(list(tv.values()), -1).astype(np.float64)
    for method in ("seuclidean", "nearest_neighbor", "zech_aslan", "szekely_rizzo", "kolmogorov_smirnov", "kldiv",
                   "mahalanobis"):
        try:
            out = analog.spatial_analogs(target, cand, method=method)
        except ValueError as e:             # frost days without spread somewhere: the reference raises too
            with pytest.raises(ValueError, match=str(e)):
                for i in range(nx):
                    for j in range(ny):
                        O.metric(method, tx, cv[:, i, j])
            continue
        assert out.dims == ("x", "y") and out.attrs["indices"] == "tg_mean,frost_days"
        got = np.asarray(out.values)
        want = np.array([[O.metric(method, tx, cv[:, i, j]) for j in range(ny)] for i in range(nx)])
        exact = method in ("nearest_neighbor", "kolmogorov_smirnov")
        if exact:
            np.testing.assert_array_equal(got, want)
        else:
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-13)
