"""CUDA implementation behind ``xclim.sdba.EmpiricalQuantileMapping``, ``QuantileDeltaMapping`` and
``DetrendedQuantileMapping`` (xsdba; PARITY UNPINNED).

``xclim.sdba`` is a shim over the third-party ``xsdba`` package (sdba.py:11) whose sources are not
part of the reference tree; the algorithm below follows its published behaviour and the reference's
call sites (tests/test_xsdba.py:21-34, 143-150): ``EQM.train(ref, hist, nquantiles=, kind=,
group="time")`` then ``.adjust(sim, interp=, extrapolation="constant")``; QDM trains the same way, DQM on
mean-normalised series.
"""
from __future__ import annotations

import numpy as np

from . import device
from .field import attrs_of, wrap_like
from .generic import _unwrap
from .options import OPTIONS

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
        r2, h2, cell_shape, other = cls._train_inputs(ref, hist, nquantiles, kind, group, kwargs)
        af, hq = device.eqm_train(r2, h2, int(nquantiles), _KINDS[kind])
        return cls(af, hq, int(nquantiles), kind, ref, cell_shape, other)

    @staticmethod
    def _train_inputs(ref, hist, nquantiles, kind, group, kwargs):
        """Validate the train options and unwrap ref, hist to (T, C): ``(r2, h2, cell_shape, other_dims)``."""
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
        return r2, h2, cell_shape, other

    @property
    def ds(self):
        """The trained dataset: ``{"af": ..., "hist_q": ...}`` with dims (quantiles, *space)."""
        q = equally_spaced_nodes(self.nquantiles).astype(np.float32)
        def wrap(t, name):
            v = t.cpu().numpy().reshape((self.nquantiles,) + self._cell_shape)
            return wrap_like(self._template, v, ("quantiles",) + self._other, coords_extra={"quantiles": q},
                             attrs={"kind": self.kind, "group": "time"}, name=name)
        return {"af": wrap(self._af, "af"), "hist_q": wrap(self._hq, "hist_q")}

    def _unwrap_sim(self, sim, interp, extrapolation, kwargs):
        """Validate the adjust options and unwrap ``sim`` to (T, C): ``(s2, other_dims, time_axis)``."""
        if interp not in _INTERP:
            raise NotImplementedError(f"interp={interp!r} is not supported (nearest, linear)")
        if extrapolation != "constant":
            raise NotImplementedError("only extrapolation='constant' is supported")
        if kwargs:
            raise NotImplementedError(f"unsupported adjust options: {sorted(kwargs)}")
        s2, cell_shape, other, ta = _unwrap(sim)
        if cell_shape != self._cell_shape:
            raise ValueError("sim grid differs from the training grid")
        return s2, other, ta

    def _wrap_series(self, sim, values, other, ta, name, attrs):
        vals = values.reshape((values.shape[0],) + self._cell_shape).cpu().numpy()
        return wrap_like(sim, vals, ("time",) + other, time=ta if ta.coord is None else ta.coord, attrs=attrs,
                         name=name)

    def adjust(self, sim, *, interp="nearest", extrapolation="constant", **kwargs):
        s2, other, ta = self._unwrap_sim(sim, interp, extrapolation, kwargs)
        scen = device.eqm_adjust(s2, self._af, self._hq, _KINDS[self.kind], _INTERP[interp])
        return self._wrap_series(sim, scen, other, ta, "scen", attrs_of(sim))


class QuantileDeltaMapping(EmpiricalQuantileMapping):
    """Quantile delta mapping bias adjustment, group="time" (xsdba ``QuantileDeltaMapping``; PARITY UNPINNED).

    ``train`` and ``.ds`` are EmpiricalQuantileMapping's.  ``adjust`` maps every value of ``sim`` through its own
    percentage rank within the cell's series (``sim_q``) instead of through ``hist_q``, so that the simulated
    change signal, trend included, is kept: ``scen = sim + af(sim_q)`` ("+") or ``sim * af(sim_q)`` ("*").  With
    ``set_options(sdba_extra_output=True)`` it returns ``{"scen": ..., "sim_q": ...}`` (``sim_q`` in float64).
    """

    def adjust(self, sim, *, interp="nearest", extrapolation="constant", **kwargs):
        s2, other, ta = self._unwrap_sim(sim, interp, extrapolation, kwargs)
        extra = bool(OPTIONS["sdba_extra_output"])
        nodes = equally_spaced_nodes(self.nquantiles).astype(np.float32)
        scen, sim_q = device.qdm_adjust(s2, self._af, nodes, _KINDS[self.kind], _INTERP[interp], want_sim_q=extra)
        out = self._wrap_series(sim, scen, other, ta, "scen", attrs_of(sim))
        if not extra:
            return out
        q = self._wrap_series(sim, sim_q, other, ta, "sim_q",
                              {"units": "", "long_name": "Percentage rank of sim within its series"})
        return {"scen": out, "sim_q": q}


def _detrend_degree(detrend):
    """xsdba's ``detrend`` argument of DQM / ``adjust``: an int is the degree of a PolyDetrend (``True`` / ``False``
    are 1 / 0, as ``isinstance(detrend, int)`` accepts them); Detrend objects are not supported."""
    if not isinstance(detrend, (int, np.integer)):
        raise NotImplementedError(f"detrend={detrend!r}: only integer polynomial degrees 0, 1 and 2 are supported")
    deg = int(detrend)
    if not 0 <= deg <= 2:
        raise NotImplementedError(f"detrend={deg}: only polynomial degrees 0, 1 and 2 are supported")
    return deg


class DetrendedQuantileMapping(EmpiricalQuantileMapping):
    """Detrended quantile mapping bias adjustment, group="time" (xsdba ``DetrendedQuantileMapping``; PARITY UNPINNED).

    ``train`` is EQM's on mean-normalised series: per cell, ``ref - mean(ref)`` and ``hist - mean(hist)`` ("+") or
    ``ref * (1 / mean(ref))`` and ``hist * (1 / mean(hist))`` ("*"); ``.ds`` adds ``scaling``, the difference ("+")
    or ratio ("*") of the two means.  ``adjust`` scales ``sim`` by ``scaling``, removes its polynomial trend of degree
    ``detrend`` (fitted over the whole series of each cell), maps the detrended values through ``hist_q -> af`` and
    puts the trend back, so that the trend of ``sim`` survives the correction.
    """

    def __init__(self, af, hist_q, scaling, nquantiles, kind, template, cell_shape, other_dims):
        super().__init__(af, hist_q, nquantiles, kind, template, cell_shape, other_dims)
        self._scaling = scaling                    # (C,) float32 device tensor

    @classmethod
    def train(cls, ref, hist, *, nquantiles=20, kind="+", group="time", **kwargs):
        r2, h2, cell_shape, other = cls._train_inputs(ref, hist, nquantiles, kind, group, kwargs)
        af, hq, scaling = device.dqm_train(r2, h2, int(nquantiles), _KINDS[kind])
        return cls(af, hq, scaling, int(nquantiles), kind, ref, cell_shape, other)

    @property
    def ds(self):
        """The trained dataset: ``af`` and ``hist_q`` (quantiles, *space) and ``scaling`` (*space)."""
        out = super().ds
        v = self._scaling.cpu().numpy().reshape(self._cell_shape)
        out["scaling"] = wrap_like(self._template, v, self._other, attrs={"kind": self.kind, "group": "time"},
                                   name="scaling")
        return out

    def adjust(self, sim, *, interp="nearest", extrapolation="constant", detrend=1, **kwargs):
        deg = _detrend_degree(detrend)
        s2, other, ta = self._unwrap_sim(sim, interp, extrapolation, kwargs)
        scen = device.dqm_adjust(s2, self._af, self._hq, self._scaling, _KINDS[self.kind], _INTERP[interp], deg)
        return self._wrap_series(sim, scen, other, ta, "scen", attrs_of(sim))
