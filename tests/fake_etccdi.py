"""TEST INFRASTRUCTURE: CPU stand-ins for the device functions of the ETCCDI percentile indices, the compound days
and the daily temperature range, on top of ``fake_device`` (same contract: numpy / oracle on CPU torch tensors,
so that the host layer can be checked without a GPU; nothing outside ``tests/`` imports it)."""
import numpy as np
import torch

import fake_device
from fake_device import OP_NAME, RED_NAME, STAT_NAME, _np, _valid
from oracle import xclim_oracle as O


def _thr(table2d, doy_index, T, per_time=False):
    t = _np(table2d)
    if doy_index is not None:
        return t[np.asarray(doy_index) - 1]
    return t if per_time else np.broadcast_to(t[:1], (T,) + t.shape[1:])


def doy_runstat(x2d, poff, doy_index, table2d, op_code, reducer_code, window, resample_before_rl=True,
                want_valid=False):
    x = _np(x2d)
    cond = O.compare(x, OP_NAME[op_code], _thr(table2d, doy_index, x.shape[0]))
    out = O.resample_and_rl(cond, bool(resample_before_rl), O.rle_statistics, poff=poff,
                            reducer=RED_NAME[reducer_code], window=int(window))
    return torch.from_numpy(np.asarray(out, dtype=np.float32)), (_valid(x, poff) if want_valid else None)


def period_sums_thr(x2d, poff, op_code, thr2d, wet, doy_index=None, per_time=False):
    x = _np(x2d)
    tp = _thr(thr2d, doy_index, x.shape[0], per_time)
    op = OP_NAME[op_code]
    over = np.where(O.compare(x, op, tp), x, 0)
    total = np.where(O.compare(x, op, float(wet)), x, 0)
    s = [np.stack([a[s:e].sum(0, dtype=np.float64) for s, e in O._groups(poff)]).astype(np.float32)
         for a in (over, total)]
    return torch.from_numpy(s[0]), torch.from_numpy(s[1])


def doy_count2(x1, x2, poff, doy_index, table1, table2, op1, op2):
    a, b = _np(x1), _np(x2)
    c = O.compare(a, OP_NAME[op1], _thr(table1, doy_index, a.shape[0])) & \
        O.compare(b, OP_NAME[op2], _thr(table2, doy_index, a.shape[0]))
    return torch.from_numpy(np.stack([c[s:e].sum(0) for s, e in O._groups(poff)]).astype(np.float32))


def period_range_stat(lo, hi, poff, stat_code, variability=False):
    d = _np(hi) - _np(lo)
    if variability:
        v = np.full_like(d, np.nan)
        v[1:] = np.abs(d[1:] - d[:-1])
        d = v
    return torch.from_numpy(O.resample_reduce(d, poff, STAT_NAME[stat_code]).astype(np.float32))


def install(monkeypatch):
    from xclim_b200 import device
    fake_device.install(monkeypatch)
    for fn in (doy_runstat, period_sums_thr, doy_count2, period_range_stat):
        monkeypatch.setattr(device, fn.__name__, fn)
