"""Missing-value masks (core/missing.py) from the fused valid counts / NaN-run kernels.

``mask[p, cell]`` is True where period ``p`` must be considered missing.  The reference computes
``valid = da.notnull()`` and resamples it once more on the CPU after every indicator
(core/indicator.py:1536-1547); here the masks come from the same streaming kernels as the indices
(SURVEY.md section 8(f).1).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, device
from .field import attrs_of
from .generic import _unwrap, _wrap_periods


def _nest(ta, subfreq, freq):
    """For every sub-period the index of the coarser period containing it (sub-periods nest)."""
    sub, big = ta.period_offsets(subfreq), ta.period_offsets(freq)
    return np.searchsorted(big, sub[:-1], side="right") - 1, len(big) - 1


def _finish(da, mask, cell_shape, other, ta, freq):
    return _wrap_periods(da, mask, cell_shape, other, ta, freq, attrs_of(da), dtype=bool)


def _valid_counts(x2d, poff):
    _, valid = device.period_count(x2d, poff, _lib.OP_NOTNAN, 0.0, want_valid=True)
    return valid


def missing_any(da, freq, src_timestep="D", **indexer):
    """core/missing.py:310-322: a period is missing if any expected step is missing.  With a
    ``select_time`` indexer only the selected steps count, on both sides of the comparison."""
    x2d, cell_shape, other, ta = _unwrap(da, indexer)
    poff = ta.period_offsets(freq)
    # expected_count (core/missing.py:64-160): a complete period of this calendar, so that a first / last
    # period the series only partly covers is missing as well
    n = torch.from_numpy(ta.expected_period_lengths(freq, **indexer).astype(np.int32)).to(x2d.device)[:, None]
    return _finish(da, _valid_counts(x2d, poff) != n, cell_shape, other, ta, freq)


def missing_pct(da, freq, tolerance, src_timestep="D", **indexer):
    """core/missing.py:453-482: missing when the fraction of missing steps reaches ``tolerance``."""
    if not 0 <= tolerance <= 1:
        raise ValueError("Options (tolerance) are invalid for missing method MissingPct.")
    x2d, cell_shape, other, ta = _unwrap(da, indexer)
    poff = ta.period_offsets(freq)
    n = torch.from_numpy(ta.expected_period_lengths(freq, **indexer).astype(np.float64)).to(x2d.device)[:, None]
    miss = (n - _valid_counts(x2d, poff).double()) / n >= tolerance
    return _finish(da, miss, cell_shape, other, ta, freq)


def at_least_n_valid(da, freq, n=20, src_timestep="D", **indexer):
    """core/missing.py:485-522: missing when fewer than ``n`` valid steps."""
    x2d, cell_shape, other, ta = _unwrap(da, indexer)
    poff = ta.period_offsets(freq)
    return _finish(da, _valid_counts(x2d, poff) < n, cell_shape, other, ta, freq)


def missing_wmo(da, freq, nm=11, nc=5, src_timestep="D", **indexer):
    """core/missing.py:394-450 (+ MissingTwoSteps :338-391): a MONTH is missing when >= nm days are
    missing or >= nc consecutive days are missing; a coarser period is missing when any of its months
    is (or when it does not hold all its months)."""
    if indexer:
        raise NotImplementedError("select_time indexers are outside the xclim_b200 hot path")
    if not (nm < 31 and nc < 31):
        raise ValueError("Options (nm, nc) are invalid for missing method MissingWMO.")
    if src_timestep != "D":
        raise ValueError(f"Input source timestep {src_timestep} is invalid for missing method MissingWMO.")
    x2d, cell_shape, other, ta = _unwrap(da)
    pm = ta.period_offsets("MS")
    # expected_count at the monthly step: the days of the complete month, so a month the series only
    # partly covers counts its absent days as missing
    nmon = torch.from_numpy(ta.expected_period_lengths("MS").astype(np.int32)).to(x2d.device)[:, None]
    missing_days = nmon - _valid_counts(x2d, pm)
    longest, _ = device.period_runstat(x2d, pm, _lib.OP_ISNAN, 0.0, _lib.RL_REDUCERS["max"], 1, True)
    miss_m = (missing_days >= nm) | (longest >= nc)
    if ta.group_ids(freq).tolist() == ta.group_ids("MS").tolist():
        return _finish(da, miss_m, cell_shape, other, ta, freq)
    parent, P = _nest(ta, "MS", freq)
    par = torch.from_numpy(parent.astype(np.int64)).to(x2d.device)
    miss = torch.zeros((P, x2d.shape[1]), dtype=torch.int32, device=x2d.device)
    miss.index_add_(0, par, miss_m.to(torch.int32))
    # second step = MissingAny over the months (:384-391): a period that does not hold all its months is
    # missing as well
    from .timeaxis import parse_offset
    mult, base, _, _ = parse_offset(freq)
    want = {"Y": 12, "Q": 3, "M": 1}[base] * mult
    short = torch.from_numpy(np.bincount(parent, minlength=P) != want).to(x2d.device)[:, None]
    return _finish(da, (miss > 0) | short, cell_shape, other, ta, freq)
