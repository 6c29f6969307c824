"""TEST INFRASTRUCTURE (like everything under oracle/): CPU restatement of quantile delta mapping (xsdba
``QuantileDeltaMapping``, group="time"; PARITY UNPINNED, the same status as EQM in xclim_oracle.py).  Its train
step is ``xclim_oracle.eqm_train`` unchanged; this module restates adjust.  The ranks come from
``scipy.stats.rankdata`` and the factor from ``scipy.interpolate.interp1d`` called as xsdba calls it, so only
xsdba's glue (the rescale of the ranks and the choice of x-table) is restated by hand.  Used by
tests/test_qdm_cpu.py, tests/test_gpu_qdm.py and bench_extra.py's CPU leg; never by the product path."""
import numpy as np

from .xclim_oracle import eqm_nodes


def qdm_rank(sim):
    """xsdba.utils.rank(sim, dim="time", pct=True): per cell, the average 1-based rank r of every valid value
    among the n valid values (bottleneck.nanrankdata == scipy.stats.rankdata(method="average") on them),
    p = r / n (xarray ``rank(pct=True)``), then ``(mx * (p - mn)) / (mx - mn)`` with mn, mx the min, max of p
    over the cell (reference CHANGELOG.rst:1043: ranks in [0, 1]).  float64, NaN where sim is NaN; a cell with
    fewer than two distinct valid values is all NaN (mx == mn)."""
    from scipy.stats import rankdata
    sim = np.asarray(sim)
    T = sim.shape[0]
    s2 = sim.reshape(T, -1)
    out = np.full(s2.shape, np.nan)
    with np.errstate(all="ignore"):
        for c in range(s2.shape[1]):
            ok = ~np.isnan(s2[:, c])
            n = int(ok.sum())
            if n == 0:
                continue
            # bottleneck ranks in float64 (recent scipy keeps float32 for float32 data; the ranks are exact in both)
            p = rankdata(s2[ok, c], method="average").astype(np.float64) / n
            mn, mx = p.min(), p.max()
            out[ok, c] = (mx * (p - mn)) / (mx - mn)
    return out.reshape(sim.shape)


def qdm_adjust(sim, af, kind="+", interp="nearest", sim_q=None):
    """QuantileDeltaMapping.adjust(group="time", extrapolation="constant"): ``sim_q = qdm_rank(sim)``; per cell
    the factor is ``scipy.interpolate.interp1d(nodes, af, kind=interp, bounds_error=False, fill_value=(first
    valid af, last valid af))`` at sim_q on the entries where af is not NaN, as xsdba's
    ``_interp_on_quantiles_1D`` calls it (float32 nodes ``eqm_nodes(nq)``, result cast to float32); then
    ``scen = sim + af_t`` or ``sim * af_t`` in float32.  ``sim_q`` (optional) replaces the computed ranks.
    Returns ``(scen, sim_q)``."""
    from scipy.interpolate import interp1d
    sim = np.asarray(sim, dtype=np.float32)
    T = sim.shape[0]
    s2 = sim.reshape(T, -1)
    af2 = np.asarray(af, dtype=np.float32).reshape(af.shape[0], -1)
    nodes = eqm_nodes(af2.shape[0]).astype(np.float32)
    q2 = (qdm_rank(s2) if sim_q is None else np.asarray(sim_q, dtype=np.float64).reshape(T, -1))
    fac = np.full(s2.shape, np.nan, dtype=np.float32)
    with np.errstate(all="ignore"):
        for c in range(s2.shape[1]):
            newx, y = q2[:, c], af2[:, c]
            mnew, mold = np.isnan(newx), np.isnan(y)
            if mnew.all() or mold.all():
                continue
            yv = y[~mold]
            f = interp1d(nodes[~mold], yv, kind=interp, bounds_error=False, fill_value=(yv[0], yv[-1]))
            fac[~mnew, c] = f(newx[~mnew])
        scen = s2 + fac if kind == "+" else s2 * fac
    return scen.astype(np.float32).reshape(sim.shape), q2.reshape(sim.shape)
