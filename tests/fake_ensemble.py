"""TEST INFRASTRUCTURE: CPU stand-ins for the ensemble entry points of ``xclim_b200.device``, built on
oracle/ensemble_oracle.py, so that the host layer of ``xclim_b200.ensembles`` (containers, names, dims, dtypes,
errors, the column walk) runs in the ``-m "not gpu"`` suite.  They prove nothing about the kernels."""
import ctypes

import numpy as np
import torch

from oracle import ensemble_oracle as E

TESTS = {0: None, 1: "abs", 2: "rel", 3: "ttest", 4: "welch-ttest", 5: "ipcc-ar6-c"}


def ens_percentiles(x2d, percentiles, alpha, beta, min_members):
    x = x2d.cpu().numpy()
    return torch.from_numpy(np.ascontiguousarray(E.percentiles(x, list(percentiles), alpha, beta, min_members)))


def ens_moments(x2d, weights, min_members):
    w = None if weights is None else weights.cpu().numpy()
    return tuple(torch.from_numpy(np.ascontiguousarray(v)) for v in E.moments(x2d.cpu().numpy(), w, min_members))


def period_reduce(x2d, poff, stat_code, transform=0, op_code=0, thr=0.0, want_valid=False):
    assert stat_code == 1 and transform == 0 and not want_valid      # the YS means of ipcc-ar6-c
    return torch.from_numpy(E.ys_annual_means(x2d.cpu().numpy()[None], poff)[0]), None


def ens_robustness(fut, ref, weights, test_code, param, strict_sign, want_pvals, ref_annual=None, ys_time=None):
    f = fut.cpu().numpy()
    r = None if ref is None else ref.cpu().numpy()
    w = None if weights is None else weights.cpu().numpy()
    t = TESTS[test_code]
    kw = {}
    if t == "abs":
        t, kw = "threshold", {"abs_thresh": param}
    elif t == "rel":
        t, kw = "threshold", {"rel_thresh": param}
    elif t == "ipcc-ar6-c":
        kw = {"refy": ref_annual.cpu().numpy(), "ys_time": ys_time.cpu().numpy()}
    elif t is not None:
        kw = {"p_change": param}
    fr, p, _ = E.robustness(f[:, 0] if r is None else f, r, t, w, strict_sign, **kw)
    frac = torch.from_numpy(np.stack([fr[k] for k in E.FRACTIONS]).reshape(7, -1))
    pv = torch.from_numpy(p.astype(np.float32).reshape(f.shape[0], -1)) if want_pvals else None
    return frac, pv


class _Lib:
    def __init__(self):
        self.boxes = []

    def xc_copy_box_async(self, dst, dst_pitch, src, src_pitch, width, rows, kind, stream):
        self.boxes.append((int(width), int(rows), int(kind)))
        for r in range(int(rows)):
            ctypes.memmove(int(dst) + r * int(dst_pitch), int(src) + r * int(src_pitch), int(width))
        return 0


def install(monkeypatch):
    """Route xclim_b200.ensembles through the stand-ins; returns the fake library (its ``boxes`` record every
    host -> device copy of the column walk)."""
    from xclim_b200 import _lib, device, ensembles
    lib = _Lib()
    for name in ("ens_percentiles", "ens_moments", "ens_robustness", "period_reduce"):
        monkeypatch.setattr(device, name, globals()[name])
    monkeypatch.setattr(device, "current_stream_ptr", lambda: 0)
    monkeypatch.setattr(ensembles, "_DEVICE", "cpu")
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(_lib, "check", lambda status: None)
    return lib
