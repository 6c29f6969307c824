"""The threshold folding rule ``xc::fold_f64`` (xclim_b200/csrc/common.cuh), compiled for the host
(tests/csrc/fold_host.cu): for every float32 x and every operator, ``x op fold(t)`` must be numpy's float64
``x op t`` (``NaN != t`` is True).  The same function folds the per-cell thresholds of the day-of-year and
array-threshold counts on the device and the scalar thresholds of every ``cmp_f64`` entry point on the host."""
import ctypes
import operator

import numpy as np
import pytest

import host_build
from xclim_b200 import _lib

#: the operators with the numpy comparison each must reproduce
OPS = {">": operator.gt, "<": operator.lt, ">=": operator.ge, "<=": operator.le, "==": operator.eq, "!=": operator.ne}


@pytest.fixture(scope="module")
def fold_lib():
    sig = (ctypes.c_int32, [ctypes.c_int32, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p])
    return host_build.load("fold", "fold_host.cu", nvcc=True, signatures={"fold_host_f64": sig})


def fold(lib, op, t):
    t = np.ascontiguousarray(t, dtype=np.float64)
    out = np.empty(t.shape, np.float32)
    assert lib.fold_host_f64(_lib.OPS[op], t.ctypes.data_as(ctypes.c_void_p), t.size,
                             out.ctypes.data_as(ctypes.c_void_p)) == 0
    return out


def edges():
    """float32 edge values (with their float32 neighbours) and float64 thresholds around them."""
    f32 = np.finfo(np.float32)
    base = np.array([0.0, 1.0, 0.1, 1.5, 278.15, 3e38, 2.0 ** -149, 2.0 ** -126 - 2.0 ** -149, 2.0 ** -126,
                     2.0 ** -125, float(f32.max), 2.0 ** 24 + 2.0], np.float32)
    base = np.concatenate([base, -base])
    with np.errstate(over="ignore"):
        up, down = np.nextafter(base, np.float32(np.inf)), np.nextafter(base, np.float32(-np.inf))
    x = np.unique(np.concatenate([base, up, down, np.array([np.inf, -np.inf, np.nan], np.float32)]))
    xd = x[np.isfinite(x)].astype(np.float64)
    t = np.concatenate([
        xd, np.nextafter(xd, np.inf), np.nextafter(xd, -np.inf),                 # float32 values, one double-ulp off
        [0.0, -0.0, 1e-300, -1e-300, 1e300, -1e300, np.inf, -np.inf, np.nan, 1e-46, -1e-46, 0.1, -0.1],
        [2.0 ** -150, -(2.0 ** -150), 3 * 2.0 ** -150, 1 + 2.0 ** -24, 1 + 3 * 2.0 ** -24],   # float32 ties
        [float(f32.max) * (1 + 2.0 ** -25), float(f32.max) * (1 + 2.0 ** -24), -float(f32.max) * (1 + 2.0 ** -24)],
    ])
    return np.append(x, np.float32(-0.0)), t   # np.unique keeps one of the two zeros


@pytest.mark.parametrize("op", list(OPS))
def test_fold_gives_the_float64_compare_for_every_float32(fold_lib, op):
    x, t = edges()
    f = fold(fold_lib, op, t)
    fn = OPS[op]
    with np.errstate(invalid="ignore"):
        got = fn(x[:, None], f[None, :])
        exp = fn(x[:, None].astype(np.float64), t[None, :])
    bad = np.argwhere(got != exp)
    assert bad.size == 0, [(float(x[i]), float(t[j]), float(f[j])) for i, j in bad[:10]]


def test_fold_keeps_float32_thresholds_and_nan(fold_lib):
    x, _ = edges()
    x = x[~np.isnan(x)]
    for op in OPS:
        np.testing.assert_array_equal(fold(fold_lib, op, x.astype(np.float64)), x)
        assert np.isnan(fold(fold_lib, op, [np.nan])[0])
    for op in ("==", "!="):
        assert np.isnan(fold(fold_lib, op, [0.1, 1e300, 1e-300])).all()
