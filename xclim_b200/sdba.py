"""CUDA implementation behind ``xclim.sdba.EmpiricalQuantileMapping`` (xsdba; PARITY UNPINNED).

``xclim.sdba`` is a shim over the third-party ``xsdba`` package (sdba.py:11) whose sources are not
part of the reference tree; the algorithm below follows its published behaviour and the reference's
call sites (tests/test_xsdba.py:21-34, 143-150): ``EQM.train(ref, hist, nquantiles=, kind=,
group="time")`` then ``.adjust(sim, interp=, extrapolation="constant")``.
"""
from __future__ import annotations

import numpy as np

from . import device
from .field import attrs_of, wrap_like
from .generic import _unwrap

_KINDS = {"+": 0, "*": 1}
_INTERP = {"nearest": 0, "linear": 1}


def equally_spaced_nodes(n):
    """xsdba.utils.equally_spaced_nodes(n, eps=None)."""
    dq = 1.0 / n / 2.0
    return np.linspace(dq, 1.0 - dq, n)


class EmpiricalQuantileMapping:
    """Empirical quantile mapping bias adjustment, group="time"."""

    def __init__(self, af, hist_q, nquantiles, kind, template, cell_shape, other_dims):
        self._af, self._hq = af, hist_q            # (nq, C) float32 device tensors
        self.nquantiles, self.kind = nquantiles, kind
        self._template, self._cell_shape, self._other = template, cell_shape, other_dims

    @classmethod
    def train(cls, ref, hist, *, nquantiles=20, kind="+", group="time", **kwargs):
        if group != "time":
            raise NotImplementedError("only group='time' is part of the xclim_b200 hot path")
        if kwargs:
            raise NotImplementedError(f"unsupported training options: {sorted(kwargs)}")
        if kind not in _KINDS:
            raise ValueError(f"kind must be '+' or '*', got {kind!r}")
        if not np.isscalar(nquantiles):
            raise NotImplementedError("explicit quantile arrays are not supported; pass an integer")
        r2, cell_shape, other, _ = _unwrap(ref)
        h2, cs2, _, _ = _unwrap(hist)
        if cs2 != cell_shape or h2.shape != r2.shape:
            raise ValueError("ref and hist must share the same shape")
        af, hq = device.eqm_train(r2, h2, int(nquantiles), _KINDS[kind])
        return cls(af, hq, int(nquantiles), kind, ref, cell_shape, other)

    @property
    def ds(self):
        """The trained dataset: ``{"af": ..., "hist_q": ...}`` with dims (quantiles, *space)."""
        q = equally_spaced_nodes(self.nquantiles).astype(np.float32)
        def wrap(t, name):
            v = t.cpu().numpy().reshape((self.nquantiles,) + self._cell_shape)
            return wrap_like(self._template, v, ("quantiles",) + self._other, coords_extra={"quantiles": q},
                             attrs={"kind": self.kind, "group": "time"}, name=name)
        return {"af": wrap(self._af, "af"), "hist_q": wrap(self._hq, "hist_q")}

    def adjust(self, sim, *, interp="nearest", extrapolation="constant", **kwargs):
        if interp not in _INTERP:
            raise NotImplementedError(f"interp={interp!r} is not supported (nearest, linear)")
        if extrapolation != "constant":
            raise NotImplementedError("only extrapolation='constant' is supported")
        if kwargs:
            raise NotImplementedError(f"unsupported adjust options: {sorted(kwargs)}")
        s2, cell_shape, other, ta = _unwrap(sim)
        if cell_shape != self._cell_shape:
            raise ValueError("sim grid differs from the training grid")
        scen = device.eqm_adjust(s2, self._af, self._hq, _KINDS[self.kind], _INTERP[interp])
        vals = scen.reshape((scen.shape[0],) + cell_shape).cpu().numpy()
        attrs = attrs_of(sim)
        return wrap_like(sim, vals, ("time",) + other, time=ta if ta.coord is None else ta.coord, attrs=attrs,
                         name="scen")
