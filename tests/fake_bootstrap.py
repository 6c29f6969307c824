"""TEST INFRASTRUCTURE: CPU stand-in for ``device.bootstrap_doy_index`` on top of ``fake_etccdi`` (same contract:
numpy / oracle on CPU torch tensors, so that the host layer can be checked without a GPU; nothing outside
``tests/`` imports it)."""
import numpy as np
import torch

import fake_etccdi
from fake_device import OP_NAME, _np
from oracle import bootstrap_oracle as B
from oracle import xclim_oracle as O


def bootstrap_doy_index(x2d, base_start, n_base_years, year_len, step_period, P, window, percentile, alpha, beta,
                        op_code, kind, run_window=1, resample_before_rl=True, floor=None, wet_total=None,
                        scratch_bytes=None):
    """The C-ABI contract of xc_bootstrap_doy_index_f32 restated with the oracle: year y's index against the table
    of the base with block y replaced by block s, averaged over s; periods without base steps NaN."""
    x = _np(x2d)
    N, L = int(n_base_years), int(year_len)
    xb = x[base_start:base_start + N * L]
    year = np.repeat(np.arange(N), L)
    doy = np.tile(np.arange(1, L + 1), N)
    sp = np.asarray(step_period)
    op = OP_NAME[op_code]
    wet = None if wet_total is None else _np(wet_total)
    out = np.full((P, x.shape[1]), np.nan, dtype=np.float32 if kind == "sum" else np.float64)
    for y in range(N):
        rows = np.nonzero(year == y)[0]
        xs = xb[rows]
        psub = sp[rows]
        periods, starts = np.unique(psub, return_index=True)
        sub = np.append(starts, L)
        vals = []
        for s_ in range(N):
            if s_ == y:
                continue
            z = xb.copy()
            z[rows] = xb[year == s_]
            tab = O.percentile_doy(z, year, doy, int(window), float(percentile), alpha, beta)[:, 0]
            if floor is not None:
                with np.errstate(invalid="ignore"):
                    tab = np.where(tab > floor, tab, floor)
            hit = O.compare(xs, op, tab)
            if kind == "count":
                vals.append(np.stack([hit[a:e].sum(0) for a, e in O._groups(sub)]))
            elif kind == "spell":
                vals.append(np.asarray(O.resample_and_rl(hit, bool(resample_before_rl), O.windowed_run_count,
                                                         int(run_window), poff=sub), dtype=np.float64))
            else:
                over = np.where(hit, xs, np.float32(0))
                s32 = np.stack([over[a:e].sum(0, dtype=np.float64) for a, e in O._groups(sub)]).astype(np.float32)
                with np.errstate(invalid="ignore", divide="ignore"):
                    vals.append(s32 / wet[periods])
        if kind == "sum":
            out[periods] = B.fraction_mean(vals)
        else:
            out[periods] = np.stack(vals).astype(np.float64).sum(0) / (N - 1)
    return torch.from_numpy(out), None


def install(monkeypatch):
    from xclim_b200 import device
    fake_etccdi.install(monkeypatch)
    monkeypatch.setattr(device, "bootstrap_doy_index", bootstrap_doy_index)
