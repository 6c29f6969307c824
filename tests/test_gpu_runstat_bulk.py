"""GPU parity of the bulk-copy run-statistic kernel (period_runstat_bulk_kernel) with the per-lane kernel and the oracle.

A scalar-threshold run statistic with runs cut at the period edges, on 4-cell-aligned data of at least one tile
(4096 cells), is fed through the bulk-copy row ring (std stays on the per-lane kernel); XCLIM_B200_RUNSTAT_V1 sends every call to the per-lane
period_runstat_kernel.  Both put every element through the same comparison, valid count and run step in time order,
so the two must agree bit for bit on every output.  The cell counts straddle the tile (W - 4 stays on the per-lane
kernel, W + 4 and 3W + 4 end on a ragged tile), the time axes end on a partial stage of rows, and the periods have
unequal lengths (months, quarters from December, a one-step period).
"""
import numpy as np
import pytest

import fake_device as F

pytestmark = pytest.mark.gpu

W = 4096
OPS = [">", "<", ">=", "<=", "==", "!=", "isnan", "notnan"]
REDUCERS = ["max", "min", "sum", "count", "mean", "std"]
THR = 1.0
MONTHS = np.array([31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31])


def _op_code(op):
    from xclim_b200 import _lib
    return {"isnan": _lib.OP_ISNAN, "notnan": _lib.OP_NOTNAN}.get(op, _lib.OPS.get(op))


def _poff(T, freq):
    """Period offsets of a 365-day calendar starting on January 1st, clipped to [0, T]."""
    years = T // 365 + 2
    if freq == "YS":
        starts = np.arange(years) * 365
    elif freq == "MS":
        starts = (np.arange(years)[:, None] * 365 + np.concatenate([[0], np.cumsum(MONTHS)[:-1]])[None, :]).ravel()
    else:   # QS-DEC: Jan-Feb, then Mar-May, Jun-Aug, Sep-Nov, Dec-Feb
        q = np.cumsum(MONTHS)[[1, 4, 7, 10]]
        starts = np.concatenate([[0], (np.arange(years)[:, None] * 365 + q[None, :]).ravel()])
    starts = starts[starts < T]
    return np.append(starts, T).astype(np.int32)


def _field(T, C, seed):
    rng = np.random.default_rng(seed)
    x = rng.gamma(0.4, 6.0, size=(T, C)).astype(np.float32)
    x[rng.random(x.shape) < 0.4] = 0.0
    x = np.round(x * 2) / 2                          # many exact ties with the threshold
    x[rng.random(x.shape) < 0.03] = np.nan
    x[:, 0] = np.nan                                 # all NaN
    x[rng.random(T) < 0.7, 1] = np.nan               # NaN-heavy
    x[:, 2] = THR                                    # constant, on the threshold
    x[:, 3] = 0.0                                    # constant, one run over every period
    x[:, -1] = np.nan                                # the last cell of the ragged tile
    x[:, -2] = 0.0
    return x.astype(np.float32)


def _sample(C):
    """Oracle cells: the special cells, both edges of every tile and of each consumer's four 1024-cell groups."""
    cells = {0, 1, 2, 3, C - 2, C - 1}
    for t0 in range(0, C, W):
        cells |= {t0, t0 + 3, min(t0 + W, C) - 4, min(t0 + W, C) - 1, t0 + 517}
        cells |= {t0 + g + d for g in (1024, 2048, 3072) for d in (-1, 0, 5)}
    return np.array(sorted(c for c in cells if 0 <= c < C))


def _both(monkeypatch, x, poff, op, red, window, want_valid):
    """(outputs of the bulk-copy dispatch, outputs of the per-lane kernel) as numpy arrays."""
    from xclim_b200 import _lib, device
    res = []
    for v1 in (False, True):
        if v1:
            monkeypatch.setenv("XCLIM_B200_RUNSTAT_V1", "1")
        else:
            monkeypatch.delenv("XCLIM_B200_RUNSTAT_V1", raising=False)
        out, valid = device.period_runstat(x, poff, _op_code(op), THR, _lib.RL_REDUCERS[red], window,
                                           resample_before_rl=True, want_valid=want_valid)
        res.append((out.cpu().numpy(), None if valid is None else valid.cpu().numpy()))
    monkeypatch.delenv("XCLIM_B200_RUNSTAT_V1", raising=False)
    return res


def _check(monkeypatch, x, xh, poff, op, red, window, want_valid, cells):
    from xclim_b200 import _lib
    (got, gval), (old, oval) = _both(monkeypatch, x, poff, op, red, window, want_valid)
    msg = f"{op} {red} w={window} valid={want_valid} P={len(poff) - 1}"
    np.testing.assert_array_equal(got.view(np.uint32), old.view(np.uint32), err_msg=msg)
    exp, eval_ = F.period_runstat(xh[:, cells], poff, _op_code(op), THR, _lib.RL_REDUCERS[red], window,
                                  want_valid=want_valid)
    if red in ("mean", "std"):
        np.testing.assert_allclose(got[:, cells], exp.numpy(), rtol=1e-5, atol=0, err_msg=msg)
    else:
        np.testing.assert_array_equal(got[:, cells], exp.numpy(), err_msg=msg)
    if want_valid:
        np.testing.assert_array_equal(gval, oval, err_msg=msg)
        np.testing.assert_array_equal(gval[:, cells], eval_.numpy(), err_msg=msg)
    else:
        assert gval is None and oval is None


@pytest.mark.parametrize("C", [W - 4, W, W + 4, 3 * W + 4])
@pytest.mark.parametrize("lat_view", [False, True], ids=["contiguous", "view"])
def test_bulk_every_op_reducer(cuda, monkeypatch, C, lat_view):
    """Every operator, reducer, window 1 and 3, with and without the valid count, on monthly periods plus a
    one-step period, T = 2 years + 4 days (not a multiple of the 4-row stage)."""
    import torch
    T = 2 * 365 + 4
    xh = _field(T, C, seed=C)
    poff = np.append(_poff(730, "MS"), [730, 731, T]).astype(np.int32)
    poff = np.unique(poff)
    assert np.any(np.diff(poff) == 1)
    if lat_view:   # a column window of a wider grid: ldx = C + 12, first cell 16-byte aligned
        buf = torch.full((T, C + 12), float("nan"), dtype=torch.float32, device=cuda)
        x = buf[:, 8:8 + C]
        x.copy_(torch.from_numpy(xh))
        assert x.stride(0) > C
    else:
        x = torch.from_numpy(xh).to(cuda)
    cells = _sample(C)
    for op in OPS:
        for red in REDUCERS:
            for window in (1, 3):
                for want_valid in (True, False):
                    _check(monkeypatch, x, xh, poff, op, red, window, want_valid, cells)


@pytest.mark.parametrize("freq", ["YS", "MS", "QS-DEC"])
def test_bulk_full_series(cuda, monkeypatch, freq):
    """30 years (T = 10950) on 3W + 4 cells: the headline statistic (dry spells, max, window 1, valid count) and the
    windowed forms, on yearly, monthly and December-quarter periods."""
    import torch
    T, C = 10950, 3 * W + 4
    xh = _field(T, C, seed=7)
    x = torch.from_numpy(xh).to(cuda)
    poff = _poff(T, freq)
    cells = _sample(C)
    for op, red, window in (("<", "max", 1), ("<", "max", 3), (">", "sum", 3), (">=", "count", 1),
                            ("<=", "mean", 3), ("<", "std", 1), ("!=", "min", 3)):
        for want_valid in (True, False):
            _check(monkeypatch, x, xh, poff, op, red, window, want_valid, cells)


def test_bulk_odd_series_length(cuda, monkeypatch):
    """T not a multiple of the stage: 10950 + 5 steps, the last yearly period 5 steps long."""
    import torch
    T, C = 10955, W + 4
    xh = _field(T, C, seed=3)
    x = torch.from_numpy(xh).to(cuda)
    poff = _poff(T, "YS")
    assert poff[-1] - poff[-2] == 5
    cells = _sample(C)
    for red in REDUCERS:
        _check(monkeypatch, x, xh, poff, "<", red, 1, True, cells)
