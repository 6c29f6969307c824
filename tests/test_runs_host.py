"""The period-edge run rule and the run-length reducers of xclim_b200/csrc/runstat.cuh (``xc::PeriodMask``,
``xc::run_step`` / ``run_close`` into ``xc::RunAcc``), compiled for the host (tests/csrc/runs_host.cu) and driven in
the order of the run-length kernels: the mask at t0 - 1, every step of the period, the steps past its end, the final
close.  Every boolean series of 12 steps, against the oracle's ``resample_and_rl`` on periods with one-step periods
and periods that leave steps before and after them, both ``resample_before_rl``, windows 1-4, all six reducers and
every accumulator form the kernels instantiate."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import xclim_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
T = 12
MASK = ((np.arange(2 ** T)[None, :] >> np.arange(T)[:, None]) & 1).astype(bool)   # (T, 4096): every series
REDUCERS = {"max": 0, "min": 1, "sum": 2, "count": 3, "mean": 4, "std": 5}
POFFS = [[0, 12], [0, 5, 12], [0, 1, 6, 7, 12], [2, 5, 9]]
FORMS = {"fixed": 0, "any": 1, "running": 2}


@pytest.fixture(scope="module")
def runs_lib():
    from xclim_b200 import _build
    out = os.path.join(tempfile.gettempdir(), f"libxclim_b200_runs_host_{os.getuid()}.so")
    src = os.path.join(HERE, "csrc", "runs_host.cu")
    deps = [src, os.path.join(ROOT, "include", "xclim_b200.h")] + \
        [os.path.join(ROOT, "xclim_b200", "csrc", h) for h in ("runstat.cuh", "common.cuh")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        cmd = [_build._nvcc(), "-O2", "-std=c++17", *_build.ARCH_FLAGS, "-Xcompiler", "-fPIC", "-shared", src,
               "-o", out]
        subprocess.run(cmd, check=True, capture_output=True, text=True)
    lib = ctypes.CDLL(out)
    lib.runs_host.restype = ctypes.c_int32
    return lib


def runs(lib, poff, before, reducer, window, form):
    poff = np.asarray(poff, np.int32)
    P, C = poff.size - 1, MASK.shape[1]
    m = np.ascontiguousarray(MASK, np.uint8)
    out = np.empty((P, C), np.float32)
    seen = np.zeros((P, T, C), np.uint8)
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731
    status = lib.runs_host(ptr(m), T, C, ptr(poff), P, int(not before), REDUCERS[reducer], window, FORMS[form],
                           ptr(out), ptr(seen))
    assert status == 0
    return out, seen.astype(bool)


def seen_from_oracle(poff, before):
    """The steps of each period's runs, from the oracle's run lengths (on the run's first step)."""
    seen = np.zeros((len(poff) - 1, T, MASK.shape[1]), bool)
    for p, (s, e) in enumerate(O._groups(np.asarray(poff))):
        d = O.rle(MASK[s:e]) if before else O.rle(MASK)[s:e]
        d = np.nan_to_num(d).astype(int)
        for k in range(d.shape[0]):
            for L in range(1, T + 1):
                seen[p, s + k:s + k + L, d[k] == L] = True
    return seen


def _check_runs(got, exp, red, msg):
    if red in ("mean", "std"):
        np.testing.assert_allclose(got, exp, rtol=1e-5, atol=0, err_msg=msg)
    else:
        np.testing.assert_array_equal(got, exp, err_msg=msg)


@pytest.mark.parametrize("before", [True, False])
@pytest.mark.parametrize("poff", POFFS, ids=["one", "5-7", "one-step", "inner"])
def test_runs_match_the_oracle(runs_lib, poff, before):
    seen_exp = seen_from_oracle(poff, before)
    for window in (1, 2, 3, 4):
        for red in REDUCERS:
            exp = O.resample_and_rl(MASK, before, O.rle_statistics, poff=np.asarray(poff), reducer=red, window=window)
            forms = ["fixed", "any"] + (["running"] if window == 1 and red in ("max", "sum", "count") else [])
            for form in forms:
                got, seen = runs(runs_lib, poff, before, red, window, form)
                msg = f"{red} w={window} {form}"
                _check_runs(got, exp, red, msg)
                np.testing.assert_array_equal(seen, seen_exp, err_msg=msg)
