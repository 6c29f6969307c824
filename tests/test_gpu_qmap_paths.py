"""Every branch of the shared quantile-mapping device code (csrc/qmap.cuh) bit for bit:

* eqm_adjust_kernel against a float32 restatement of its arithmetic (slope, midpoint, end factors), on nodes,
  midpoints and their float32 neighbours, out of range, +-inf, NaN, +-0, degenerate and NaN tables, a position-table
  bin that holds most nodes (the scan past its two unrolled steps), and grid edges;
* EQM train through the 32-cell layout, the 16-cell layout and the one-cell kernel against the oracle;
* the interp1d factor of qdm_apply_kernel and dqm_adjust_kernel against the oracles fed the kernels' own ranks and
  trend coefficients: NaN table entries, one valid entry and none, duplicate keys, many keys in one position-table
  bin, values exactly on a key or a nearest bound."""
import numpy as np
import pytest

from oracle import dqm_oracle as D
from oracle import qdm_oracle as Q
from oracle import xclim_oracle as O

pytestmark = pytest.mark.gpu

F32 = np.float32
KIND = {"+": 0, "*": 1}
INTERP = {"nearest": 0, "linear": 1}


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits_equal(got, exp, msg):
    """float32 arrays equal bit for bit (signed zeros included), any NaN matching any NaN"""
    got, exp = (np.where(np.isnan(a), F32(np.nan), a).astype(F32).view(np.uint32) for a in (got, exp))
    np.testing.assert_array_equal(got, exp, err_msg=msg)


# ---------------------------------------------------------------------------------------------------- EQM adjust
def eqm_adjust_f32(sim, af, hq, kind, interp):
    """eqm_adjust_kernel's arithmetic in numpy float32: any NaN in a cell's table gives NaN; x <= hq[0] -> af[0],
    x >= hq[-1] -> af[-1]; else idx = #{hq < x} in [1, nq - 1] and linear slope[idx] * (x - x0) + y0 with
    slope[j] = (af[j] - af[j-1]) / (hq[j] - hq[j-1]), or nearest y0 when x <= (x0 + x1) * 0.5, else y1."""
    T, C = sim.shape
    nq = hq.shape[0]
    out = np.full((T, C), np.nan, F32)
    with np.errstate(all="ignore"):
        for c in range(C):
            h, a, x = hq[:, c], af[:, c], sim[:, c]
            if np.isnan(h).any() or np.isnan(a).any():
                continue
            idx = np.clip((h[None, :] < x[:, None]).sum(axis=1), 1, nq - 1)
            x0, y0, x1, y1 = h[idx - 1], a[idx - 1], h[idx], a[idx]
            if interp == "linear":
                slope = (a[1:] - a[:-1]) / (h[1:] - h[:-1])
                f = slope[idx - 1] * (x - x0) + y0
            else:
                f = np.where(x <= (x0 + x1) * F32(0.5), y0, y1)
            f = np.where(x >= h[-1], a[-1], f)
            f = np.where(x <= h[0], a[0], f)
            f = np.where(np.isnan(x), F32(np.nan), f).astype(F32)
            out[:, c] = x + f if kind == "+" else x * f
    return out


def _eqm_tables(rng, nq, C):
    """(nq, C) hist_q and af: sorted random columns and one hostile table per column 0 .. 8."""
    hq = np.sort(rng.standard_normal((nq, C)) * 8, axis=0).astype(F32)
    af = rng.standard_normal((nq, C)).astype(F32)
    hq[:, 0] = np.round(hq[:, 0])                                     # duplicate nodes
    af[nq // 2:, 0] = af[nq // 2, 0]                                  # a flat stretch
    hq[:, 1] = F32(2.5)                                               # constant: position-table scale 0
    hq[0, 2], hq[-1, 2] = -np.inf, np.inf                            # infinite range: scale 0 too
    hq[:, 3] = np.append(np.linspace(0, 1e-3, nq - 1), 100.0)         # all but one node in table bin 0
    hq[:, 4] = np.append(-100.0, np.linspace(0, 1e-3, nq - 1))        # ... in the top bin
    hq[nq // 2, 5] = np.nan                                           # NaN in hist_q: the cell is NaN
    af[-1, 6] = np.nan                                                # NaN in af: the cell is NaN
    hq[:, 7] = (hq[:, 7] * F32(1e37)).astype(F32)                     # huge nodes: midpoints overflow
    hq[:, 8] = np.sort(np.where(np.arange(nq) % 2 == 0, F32(-0.0), F32(0.0)) + np.arange(nq) // 2).astype(F32)
    return hq, af


def _eqm_sim(rng, T, hq):
    """(T, C): per column out-of-range values, +-inf, NaN, +-0, the nodes, the midpoints and their float32
    neighbours (as many as T holds), then uniform values in the range; shuffled."""
    nq, C = hq.shape
    sim = np.empty((T, C), F32)
    with np.errstate(all="ignore"):
        for c in range(C):
            h = hq[:, c]
            mid = (h[:-1] + h[1:]) * F32(0.5)
            pts = np.concatenate([h, mid])
            pts = np.concatenate([pts, np.nextafter(pts, F32(np.inf)), np.nextafter(pts, F32(-np.inf))])
            fin = h[np.isfinite(h)]
            lo, hi = (fin.min(), fin.max()) if fin.size else (F32(0), F32(1))
            extra = np.array([lo - 1, hi + 1, np.inf, -np.inf, np.nan, 0.0, -0.0], F32)
            fill = rng.uniform(lo, hi if hi > lo else lo + 1, T).astype(F32)
            col = np.concatenate([extra, pts, fill])[:T]
            sim[:, c] = rng.permutation(col)
    return sim


@pytest.mark.parametrize("nq", [2, 3, 20, 64])
@pytest.mark.parametrize("kind,interp", [("+", "linear"), ("+", "nearest"), ("*", "linear"), ("*", "nearest")])
@pytest.mark.parametrize("T", [1003, 50])     # T not a multiple of the 16 rows in flight; T below the 64-row split
def test_eqm_adjust_bit_identical(cuda, nq, kind, interp, T):
    """eqm_adjust_kernel: position table (qmap::PosTable), scan, slope / midpoint / end factors; C = 150 (not a
    multiple of 128) read from a column slice (ldx > C)."""
    from xclim_b200 import device
    rng = np.random.default_rng(90 + nq + T)
    C = 150
    hq, af = _eqm_tables(rng, nq, C)
    sim = _eqm_sim(rng, T, hq)
    big = np.full((T, C + 7), np.nan, F32)
    big[:, 3:3 + C] = sim
    d = _cuda(big)[:, 3:3 + C]
    assert d.stride(0) == C + 7
    scen = device.eqm_adjust(d, _cuda(af), _cuda(hq), KIND[kind], INTERP[interp]).cpu().numpy()
    _bits_equal(scen, eqm_adjust_f32(sim, af, hq, kind, interp), f"nq={nq} {kind} {interp} T={T}")


# ---------------------------------------------------------------------------------------------------- EQM train
def _train_data(rng, T, C, kind):
    if kind == "+":
        ref, hist = 285 + 6 * rng.standard_normal((T, C)), 286.5 + 7 * rng.standard_normal((T, C))
    else:
        ref, hist = 0.2 + rng.gamma(0.8, 4.0, (T, C)), 0.2 + rng.gamma(0.7, 5.0, (T, C))
    ref, hist = ref.astype(F32), hist.astype(F32)
    hist[rng.random(hist.shape) < 0.01] = np.nan
    hist[:, 1] = np.round(hist[:, 1])                                   # ties
    ref[:, 0] = np.nan                                                  # untrainable cell
    return ref, hist


@pytest.mark.parametrize("nq", [2, 20, 64])
@pytest.mark.parametrize("kind", ["+", "*"])
def test_eqm_train_layouts_bit_identical(cuda, kind, nq, monkeypatch):
    """eqm_train_group_kernel with 32 cells per CTA (C = 96; nq = 64 does not fit and takes 16), with 16 cells
    per CTA (C = 80) and eqm_train_kernel alone, each against the oracle bit for bit."""
    from xclim_b200 import device
    rng = np.random.default_rng(95 + nq)
    ref, hist = _train_data(rng, 1500, 96, kind)
    e_af, e_hq = O.eqm_train(ref, hist, nq, kind)
    monkeypatch.delenv("XCLIM_B200_EQM_V1", raising=False)
    for C, label in ((96, "32-cell"), (80, "16-cell")):
        af, hq = device.eqm_train(_cuda(ref[:, :C]), _cuda(hist[:, :C]), nq, KIND[kind])
        _bits_equal(hq.cpu().numpy(), e_hq[:, :C], f"{label} hist_q")
        _bits_equal(af.cpu().numpy(), e_af[:, :C], f"{label} af")
    monkeypatch.setenv("XCLIM_B200_EQM_V1", "1")
    af, hq = device.eqm_train(_cuda(ref), _cuda(hist), nq, KIND[kind])
    _bits_equal(hq.cpu().numpy(), e_hq, "one-cell hist_q")
    _bits_equal(af.cpu().numpy(), e_af, "one-cell af")


# ---------------------------------------------------------------------------------------------------- QDM, DQM
def _factor_tables(rng, nq, C):
    """(nq, C) af with NaN entries (columns 0, 1), one valid entry (2), none (3); the rest random."""
    af = (rng.standard_normal((nq, C)) * 0.5).astype(F32)
    af[nq // 2, 0] = np.nan
    af[[0, -1], 1] = np.nan
    af[:-1, 2] = np.nan
    af[:, 3] = np.nan
    return af


@pytest.mark.parametrize("nq", [2, 4, 20])
@pytest.mark.parametrize("kind,interp", [("+", "linear"), ("+", "nearest"), ("*", "linear"), ("*", "nearest")])
def test_qdm_factor_bit_identical(cuda, nq, kind, interp):
    """qdm_apply_kernel's interp1d (qmap::interp1d_edges, linear_two_weight, nearest_bound) against the oracle fed
    the kernel's sim_q.  T = 33 distinct values per cell: sim_q hits the nodes and nearest bounds of nq = 2 and 4
    exactly."""
    from xclim_b200 import device
    rng = np.random.default_rng(97 + nq)
    T, C = 33, 40
    sim = np.stack([rng.permutation(np.arange(1, T + 1)) for _ in range(C)], axis=1).astype(F32)
    sim[rng.random(sim.shape) < 0.05] = np.nan
    sim[:, 4:8] = np.arange(1, T + 1, dtype=F32)[:, None]             # no NaN: sim_q exactly on the grid
    af = _factor_tables(rng, nq, C)
    scen, q = device.qdm_adjust(_cuda(sim), _cuda(af), O.eqm_nodes(nq).astype(F32), KIND[kind], INTERP[interp],
                                want_sim_q=True)
    q = q.cpu().numpy()
    exp, _ = Q.qdm_adjust(sim, af, kind, interp, sim_q=q)
    _bits_equal(scen.cpu().numpy(), exp, f"nq={nq} {kind} {interp}")
    if nq in (2, 4):
        nodes = O.eqm_nodes(nq).astype(F32).astype(np.float64)
        bounds = (nodes[:-1] / 2 + nodes[1:] / 2)
        assert np.isin(q[:, 4], nodes).any() and np.isin(q[:, 4], bounds).any()


@pytest.mark.parametrize("kind,interp", [("+", "linear"), ("+", "nearest"), ("*", "linear"), ("*", "nearest")])
def test_dqm_factor_bit_identical(cuda, kind, interp):
    """dqm_adjust_kernel's interp1d and position table (qmap::PosTable<double>) against the oracle fed the kernel's
    trend coefficients.  Columns 10, 11 are constant 2.0 at degree 0, so d is exactly 0 ("+") or 1 ("*"): on a key
    of column 10 and on a nearest bound of column 11."""
    from xclim_b200 import device
    rng = np.random.default_rng(99)
    T, C, nq = 40, 48, 8
    sim = (rng.standard_normal((T, C)) * 3).astype(F32)
    sim[rng.random(sim.shape) < 0.05] = np.nan
    hq = np.sort(rng.standard_normal((nq, C)) * 3, axis=0).astype(F32)
    af = _factor_tables(rng, nq, C)
    hq[2, 4] = np.nan                                                   # NaN in hist_q
    hq[:, 5] = np.nan                                                   # no valid entry through hist_q
    hq[:, 6] = np.round(hq[:, 6])                                       # duplicate keys
    hq[:, 7] = np.append(np.linspace(0, 1e-3, nq - 1), 50.0)            # all but one key in table bin 0
    hq[:, 8] = np.append(-50.0, np.linspace(0, 1e-3, nq - 1))           # ... in the top bin
    sim[:, 10:12] = 2.0
    hq[:, 10] = [-1, 0, 1, 3, 4, 5, 6, 7]                               # keys 0 and 1
    hq[:, 11] = [-1, 1, 3, 5, 6, 7, 8, 9]                               # nearest bounds 0 and 2, key 1
    sc = np.zeros(C, F32) if kind == "+" else np.ones(C, F32)
    scen, coef = device.dqm_adjust(_cuda(sim), _cuda(af), _cuda(hq), _cuda(sc), KIND[kind], INTERP[interp], 0,
                                   want_coef=True)
    coef = coef.cpu().numpy()
    assert (coef[0, 10:12] == 2.0).all()
    exp = D.dqm_adjust(sim, af, hq, sc, kind, interp, detrend=0, coef=coef)
    _bits_equal(scen.cpu().numpy(), exp, f"{kind} {interp}")
