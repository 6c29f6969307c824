"""The host build of the bootstrap mask reducer (xclim_b200/csrc/bootstrap_reduce_core.cuh, through
tests/csrc/bootstrap_reduce_host.cu) against the oracle's reduction of the same masks: days over the threshold,
windowed_run_count with both period-edge rules (resample_and_rl on year y's own slice) and the fraction with the
float64 mean of the non-NaN float32 terms."""
import ctypes

import numpy as np
import pytest

import host_build
from oracle import bootstrap_oracle as B
from oracle import xclim_oracle as O

RED = {"count": 0, "spell": 1, "sum": 2}


def _lib():
    vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32
    sig = (None, [i32, vp, i64, i32, i32, i32, vp, i32, i32, vp, i64, vp, vp])
    return host_build.load("boot_reduce", "bootstrap_reduce_host.cu", nvcc=True,
                           signatures={"boot_reduce_host": sig})


def _case(seed, N, L, C, ppy):
    rng = np.random.default_rng(seed)
    # runs of every length: a two-state chain with long stays, so that periods end inside runs
    bits = np.zeros((N * (N - 1), L, C), bool)
    state = rng.random((N * (N - 1), C)) < 0.5
    for d in range(L):
        flip = rng.random(state.shape) < 0.18
        state = state ^ flip
        bits[:, d] = state
    x = rng.gamma(0.8, 4.0, (N * L, C)).astype(np.float32)
    u = rng.random(x.shape)
    x[u < 0.03] = np.nan
    x[(u > 0.5) & (u < 0.51)] = np.inf
    x[(u > 0.6) & (u < 0.605)] = -np.inf
    edges = np.sort(rng.choice(np.arange(1, L), ppy - 1, replace=False)) if ppy > 1 else np.array([], int)
    per_year = np.zeros(L, np.int32)
    per_year[edges] = 1
    per_year = np.cumsum(per_year).astype(np.int32)
    sp = np.concatenate([per_year + y * ppy for y in range(N)]).astype(np.int32)
    wet = rng.gamma(2.0, 20.0, (N * ppy, C)).astype(np.float32)
    wet[rng.random(wet.shape) < 0.05] = 0.0
    return bits, x, sp, wet


def _pack(bits, L):
    pairs, _, C = bits.shape
    Wd = (L + 31) // 32
    pad = np.zeros((pairs, Wd * 32, C), np.uint32)
    pad[:, :L] = bits
    w = (pad.reshape(pairs, Wd, 32, C) << np.arange(32, dtype=np.uint32)[None, None, :, None]).sum(2)
    return np.ascontiguousarray(w.astype(np.uint32)), Wd


def _oracle(kind, bits, x, sp, wet, N, L, window, before):
    P, C = wet.shape
    out = np.full((P, C), np.nan, np.float32 if kind == "sum" else np.float64)
    for y in range(N):
        psub = sp[y * L:(y + 1) * L]
        periods, starts = np.unique(psub, return_index=True)
        sub = np.append(starts, L)
        xs = x[y * L:(y + 1) * L]
        vals = []
        for s in range(N):
            if s == y:
                continue
            m = bits[y * (N - 1) + (s if s < y else s - 1)]
            if kind == "count":
                vals.append(np.stack([m[a:e].sum(0) for a, e in O._groups(sub)]))
            elif kind == "spell":
                vals.append(np.asarray(O.resample_and_rl(m, before, O.windowed_run_count, window, poff=sub),
                                       np.float64))
            else:
                over = np.where(m, xs, np.float32(0))
                s32 = np.stack([over[a:e].sum(0, dtype=np.float64) for a, e in O._groups(sub)]).astype(np.float32)
                with np.errstate(invalid="ignore", divide="ignore"):
                    vals.append(s32 / wet[periods])
        out[periods] = B.fraction_mean(vals) if kind == "sum" else np.stack(vals).astype(np.float64).sum(0) / (N - 1)
    return out


@pytest.mark.parametrize("kind,window,before", [("count", 1, True), ("sum", 1, True)] +
                         [("spell", w, b) for w in range(1, 9) for b in (True, False)])
@pytest.mark.parametrize("N,L,ppy", [(3, 40, 4), (4, 70, 1), (5, 37, 3)])
def test_reducer_equals_oracle(kind, window, before, N, L, ppy):
    C = 9
    bits, x, sp, wet = _case(N * 100 + L + window, N, L, C, ppy)
    words, Wd = _pack(bits, L)
    out = np.zeros(wet.shape, np.float32 if kind == "sum" else np.float64)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    _lib().boot_reduce_host(RED[kind], p(words), C, Wd, N, L, p(sp), window, int(not before), p(x), C, p(wet), p(out))
    exp = _oracle(kind, bits, x, sp, wet, N, L, window, before)
    np.testing.assert_array_equal(out, exp)
    if kind == "sum":
        assert np.isnan(out).any() and np.isfinite(out).any()
