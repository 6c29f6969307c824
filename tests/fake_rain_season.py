"""TEST INFRASTRUCTURE: a CPU stand-in for ``device.rain_season`` on top of ``fake_device`` (same contract: the oracle
on CPU torch tensors, so that the host layer can be checked without a GPU; nothing outside ``tests/`` imports it).
The date selections come from the kernel's mask bits; the rest is the oracle's period function."""
import numpy as np
import torch

import fake_device
from fake_device import _np
from oracle import rain_season_oracle as R
from xclim_b200 import _lib

METHOD_NAME = {v: k for k, v in _lib.RS_METHODS.items()}


def rain_season(x2d, poff, mask, scale, thr_wet, window_wet, window_not_dry, thr_dry_start, window_dry_start,
                method_dry_start, thr_dry_end, window_dry_end, method_dry_end):
    p = R.params32(dict(thresh_wet_start=thr_wet, window_wet_start=window_wet, window_not_dry_start=window_not_dry,
                        thresh_dry_start=thr_dry_start, window_dry_start=window_dry_start,
                        method_dry_start=METHOD_NAME[method_dry_start], thresh_dry_end=thr_dry_end,
                        window_dry_end=window_dry_end, method_dry_end=METHOD_NAME[method_dry_end]))
    pram = _np(x2d).astype(np.float32) * np.float32(scale)
    mask = np.asarray(mask)
    out = []
    for a, b in zip(poff[:-1], poff[1:]):
        m = mask[a:b]
        s, e, _ = R.period(pram[a:b], (m & _lib.RS_PRE) > 0, (m & _lib.RS_START) > 0, (m & _lib.RS_END) > 0, p)
        out.append([np.where(np.isnan(v), -1, v).astype(np.int32) for v in (s, e)])
    return tuple(torch.from_numpy(np.stack([o[k] for o in out])) for k in (0, 1))


def install(monkeypatch):
    from xclim_b200 import device
    fake_device.install(monkeypatch)
    monkeypatch.setattr(device, "rain_season", rain_season)
