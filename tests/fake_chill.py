"""TEST INFRASTRUCTURE: CPU stand-ins for ``device.chill_daily``, ``device.chill_hourly`` and
``device.hourly_temperature`` on top of ``fake_device`` (same contract, on CPU torch tensors), so that the host layer
can be checked without a GPU; nothing outside ``tests/`` imports it.  They run the host build of chill_core.cuh,
which ``test_chill_cpu.py`` checks against the oracle."""
import numpy as np
import torch

import chill_host_build as H
import fake_device
from fake_device import _np


def _mask(m):
    return None if m is None else np.asarray(m, np.uint8)


def _out(what, cp, cu, valid, want_valid):
    from xclim_b200 import _lib
    t = torch.from_numpy
    return (t(cp) if what & _lib.CHILL_PORTIONS else None, t(cu) if what & _lib.CHILL_UNITS else None,
            t(valid) if want_valid else None)


def chill_daily(tasmin, tasmax, weights, lat_index, poff, day_mask, to_k, to_c, what, want_valid=False):
    cp, cu, valid = H.chill(poff, _mask(day_mask), to_k, to_c, what, tasmin=_np(tasmin), tasmax=_np(tasmax),
                            weights=_np(weights), lat_index=_np(lat_index))
    return _out(what, cp, cu, valid, want_valid)


def chill_hourly(x2d, poff, day_mask, to_k, to_c, what, want_valid=False):
    cp, cu, valid = H.chill(poff, _mask(day_mask), to_k, to_c, what, hourly=_np(x2d))
    return _out(what, cp, cu, valid, want_valid)


def hourly_temperature(tasmin, tasmax, weights, lat_index):
    return torch.from_numpy(H.hourly_temperature(_np(tasmin), _np(tasmax), _np(weights), _np(lat_index)))


def to_time_cell_f64(values, time_axis):
    a = np.ascontiguousarray(np.moveaxis(_np(values), time_axis, 0), np.float64)
    return torch.from_numpy(a.reshape(a.shape[0], -1)), tuple(a.shape[1:])


def install(monkeypatch):
    from xclim_b200 import device
    fake_device.install(monkeypatch)
    for fn in (chill_daily, chill_hourly, hourly_temperature, to_time_cell_f64):
        monkeypatch.setattr(device, fn.__name__, fn)
