"""Quantile delta mapping on the GPU against the oracle (oracle/qdm_oracle.py: qdm_rank, qdm_adjust; PARITY UNPINNED
against xsdba itself): sim_q and scen bit for bit.
Covers both kinds and interpolations, nq from 2 to 200, hostile data (ties, signed zeros, NaN, degenerate cells,
infinities, +-3e38, NaN inside af), the layouts (short and long series, partial 32-cell tiles, column slices, cell
chunks) and a headline-size sample."""
import numpy as np
import pytest

from oracle import qdm_oracle as Q
from oracle import xclim_oracle as O
from xb_helpers import make_field

pytestmark = pytest.mark.gpu

KIND = {"+": 0, "*": 1}
INTERP = {"nearest": 0, "linear": 1}


def _gpu(sim_dev, af, kind, interp, workspace_bytes=None):
    import torch
    from xclim_b200 import device
    nodes = O.eqm_nodes(af.shape[0]).astype(np.float32)
    scen, q = device.qdm_adjust(sim_dev, torch.from_numpy(np.ascontiguousarray(af)).cuda(), nodes, KIND[kind],
                                INTERP[interp], want_sim_q=True, workspace_bytes=workspace_bytes)
    return scen.cpu().numpy(), q.cpu().numpy()


def _compare(sim, af, kind, interp, scen, q, label):
    exp_scen, exp_q = Q.qdm_adjust(sim, af, kind, interp)
    assert q.dtype == np.float64 and scen.dtype == np.float32
    np.testing.assert_array_equal(q, exp_q, err_msg=f"sim_q {label}")
    np.testing.assert_array_equal(scen, exp_scen, err_msg=f"scen {label}")


def _pr(rng, T, C, step=0.1):
    x = rng.gamma(0.5, 6.0, size=(T, C)).astype(np.float32)
    x[rng.random(x.shape) < 0.45] = 0.0
    return (np.round(x / step) * step).astype(np.float32)


@pytest.mark.parametrize("nq", [2, 20, 64])
@pytest.mark.parametrize("kind,interp", [("+", "linear"), ("+", "nearest"), ("*", "linear"), ("*", "nearest")])
def test_qdm_train_adjust(cuda, kind, interp, nq):
    import xclim_b200
    from xclim_b200 import sdba
    rng = np.random.default_rng(61)
    T, shape = 1500, (3, 37)                     # 111 cells: a partial 32-cell tile
    if kind == "+":
        ref = (285 + 6 * rng.standard_normal((T,) + shape)).astype(np.float32)
        hist = (286.5 + 7 * rng.standard_normal((T,) + shape)).astype(np.float32)
        sim = (288.5 + 7 * rng.standard_normal((T + 400,) + shape) + np.linspace(0, 4, T + 400)[:, None, None])
        units = "K"
    else:
        ref = 0.2 + rng.gamma(0.8, 4.0, (T,) + shape)
        hist = 0.2 + rng.gamma(0.7, 5.0, (T,) + shape)
        sim = 0.2 + rng.gamma(0.7, 5.5, (T + 400,) + shape)
        units = "mm/d"
    ref, hist, sim = (a.astype(np.float32) for a in (ref, hist, sim))
    hist[rng.random(hist.shape) < 0.01] = np.nan
    sim[rng.random(sim.shape) < 0.01] = np.nan
    ref[:, 0, 0] = np.nan                          # untrainable cell: af all NaN -> scen NaN
    f = lambda a: make_field(a, "1981-01-01", calendar="noleap", units=units)  # noqa: E731
    qdm = sdba.QuantileDeltaMapping.train(f(ref), f(hist), nquantiles=nq, kind=kind, group="time")
    with xclim_b200.set_options(sdba_extra_output=True):
        out = qdm.adjust(f(sim), interp=interp, extrapolation="constant")
    scen, q = out["scen"].values, out["sim_q"].values
    assert scen.shape == sim.shape and q.shape == sim.shape and out["scen"].attrs["units"] == units
    _compare(sim, qdm.ds["af"].values, kind, interp, scen, q, f"train nq={nq} {kind} {interp}")
    plain = qdm.adjust(f(sim), interp=interp)
    np.testing.assert_array_equal(plain.values, scen)


def _hostile(rng, T, nq):
    """(T, C) sim with one hostile pattern per cell and a matching (nq, C) af."""
    C = 45
    sim = (280 + 9 * rng.standard_normal((T, C))).astype(np.float32)
    sim[:, 0:6] = _pr(rng, T, 6)                                          # quantised precipitation, ~45 % zeros
    sim[:, 6] = np.where(rng.random(T) < 0.5, np.float32(-0.0), np.float32(0.0))
    sim[rng.random(T) < 0.3, 6] = 1.5                                     # -0.0 next to +0.0, one more value
    sim[rng.random(T) < 0.2, 7] = np.nan                                  # scattered NaN
    sim[:, 8] = np.nan                                                    # all NaN
    sim[:, 9] = np.nan
    sim[T // 2, 9] = 4.0                                                  # one valid value
    sim[:, 10] = 3.0                                                      # constant
    sim[:, 11] = -2.0
    sim[rng.random(T) < 0.3, 11] = np.nan                                 # constant with NaN
    sim[:, 12] = np.where(rng.random(T) < 0.3, 1.0, 2.0)                  # two values
    u = rng.random(T)
    sim[u < 0.05, 13] = np.inf                                            # +-inf among ordinary values
    sim[u > 0.97, 13] = -np.inf
    sim[u < 0.02, 14] = np.float32(3e38)                                  # +-3e38: a stretched range
    sim[u > 0.99, 14] = np.float32(-3e38)
    sim[:, 15] = np.where(u < 0.5, np.float32(-3e38), np.float32(3e38))
    sim[u < 0.1, 15] = np.inf
    sim[:, 16] = np.where(u < 0.4, -np.inf, np.inf)                       # infinities only
    sim[:, 17] = rng.exponential(5.0, T).astype(np.float32)              # continuous, skewed
    sim[:, 18] = (np.arange(T) % 7).astype(np.float32)                    # seven values, heavy ties
    sim[:, 19] = np.float32(1.0) + (rng.integers(0, 3, T) * np.float32(1.2e-7)).astype(np.float32)   # ulp apart
    af = np.cumsum(rng.random((nq, C)) * 0.5, axis=0).astype(np.float32) - 0.2 * nq
    if nq > 2:
        af[1, 20] = np.nan                                                # NaN entries inside af
        af[nq // 2:nq // 2 + 3, 21] = np.nan
        af[[0, -1], 23] = np.nan                                          # first and last NaN
        af[:-1, 24] = np.nan                                              # one valid entry
    af[:, 22] = np.nan                                                    # all NaN
    af[0, 25] = -np.inf                                                   # infinite factors
    af[-1, 26] = np.inf
    return sim, af


@pytest.mark.parametrize("nq", [2, 200])
@pytest.mark.parametrize("kind,interp", [("+", "linear"), ("+", "nearest"), ("*", "linear"), ("*", "nearest")])
def test_qdm_hostile_data(cuda, kind, interp, nq):
    import torch
    rng = np.random.default_rng(62 + nq)
    sim, af = _hostile(rng, 3000, nq)
    scen, q = _gpu(torch.from_numpy(sim).cuda(), af, kind, interp)
    _compare(sim, af, kind, interp, scen, q, f"hostile nq={nq} {kind} {interp}")
    assert np.isnan(q[:, [8, 9, 10, 11]]).all() and np.isnan(scen[:, [8, 9, 10, 11, 22]]).all()
    assert np.array_equal(q[:, 6] == q[:, 6].min(), sim[:, 6] == 0)     # both zeros in the bottom tie group


@pytest.mark.parametrize("T", [1, 2, 40, 10950, 32768])
def test_qdm_layouts(cuda, T):
    """Series lengths, a partial last tile, a column slice (ldx > C) and cell chunks forced by the smallest
    workspace: all against the oracle, chunked == unchunked bit for bit."""
    import torch
    from xclim_b200 import _lib, device
    rng = np.random.default_rng(63)
    C, nq = 70, 20
    big = (285 + 8 * rng.standard_normal((T, C + 9))).astype(np.float32)
    big[rng.random(big.shape) < 0.02] = np.nan
    big[:, 5] = np.round(big[:, 5])
    sim = big[:, 3:3 + C]
    af = np.cumsum(rng.random((nq, C)), axis=0).astype(np.float32) - 10
    d = torch.from_numpy(big).cuda()[:, 3:3 + C]
    assert d.stride(0) == C + 9
    scen, q = _gpu(d, af, "+", "linear")
    _compare(sim, af, "+", "linear", scen, q, f"T={T} slice")
    ws_min = int(_lib.load().xc_qdm_adjust_workspace_bytes(T, 32))
    scen_c, q_c = _gpu(d, af, "+", "linear", workspace_bytes=ws_min)        # three chunks of <= 32 cells
    np.testing.assert_array_equal(scen_c, scen)
    np.testing.assert_array_equal(q_c, q)
    if T == 32768:
        x = torch.zeros((T + 1, 4), device="cuda")
        with pytest.raises(NotImplementedError, match="32768"):
            device.qdm_adjust(x, torch.zeros((nq, 4), device="cuda"), O.eqm_nodes(nq).astype(np.float32), 0, 1)


def test_qdm_headline_sample(cuda):
    """The headline series (10950 days of synthetic tasmax, 1440 cells per lat row) on a lat sub-tile sized from
    the free device memory; 4096 sampled cells and the last 256 against the oracle."""
    import torch
    from xclim_b200 import device
    T, X = 10950, 1440
    free = torch.cuda.mem_get_info()[0]
    rows = int(max(4, min(180, free * 0.4 // (X * T * 26))))                 # ref, hist, sim, scen, sim_q, scratch
    C = rows * X
    ref = device.synth(T, C, kind=1, seed=3, cells_per_lat=X, n_lat_global=rows)
    hist = device.synth(T, C, kind=1, seed=5, cells_per_lat=X, n_lat_global=rows)
    af, _ = device.eqm_train(ref, hist, 20, 0)
    del ref, hist
    sim = device.synth(T, C, kind=1, seed=7, cells_per_lat=X, n_lat_global=rows)
    scen, q = device.qdm_adjust(sim, af, O.eqm_nodes(20).astype(np.float32), 0, 1, want_sim_q=True)
    rng = np.random.default_rng(64)
    cells = np.unique(np.concatenate([rng.choice(C - 256, 4096, replace=False), np.arange(C - 256, C)]))
    idx = torch.from_numpy(cells).cuda()
    s, a = sim[:, idx].cpu().numpy(), af[:, idx].cpu().numpy()
    _compare(s, a, "+", "linear", scen[:, idx].cpu().numpy(), q[:, idx].cpu().numpy(), f"headline {rows} rows")


@pytest.mark.parametrize("kind", ["+", "*"])
@pytest.mark.parametrize("interp", ["linear", "nearest"])
def test_qdm_preserves_ranks(cuda, kind, interp):
    """QDM keeps the order of sim within a cell (tests/test_xsdba.py:112-155 spirit): with a non-decreasing af,
    scen is non-decreasing in sim ("+"; "*" on positive data), and sim_q orders like sim."""
    import torch
    rng = np.random.default_rng(65)
    T, C, nq = 4000, 64, 30
    # on a 1/64 grid for "*": distinct values lie far more than the 1-ulp rounding of af_t at a node apart
    sim = (np.round((0.5 + rng.gamma(2.0, 3.0, (T, C))) * 64) / 64).astype(np.float32) if kind == "*" else \
        (285 + 8 * rng.standard_normal((T, C))).astype(np.float32)
    sim[:, 3] = np.round(sim[:, 3])                                          # ties
    af = np.cumsum(rng.random((nq, C)) * 0.1, axis=0).astype(np.float32) + (0.5 if kind == "*" else -1.0)
    scen, q = _gpu(torch.from_numpy(sim).cuda(), af, kind, interp)
    for c in range(C):
        o = np.argsort(sim[:, c], kind="stable")
        assert (np.diff(scen[o, c]) >= 0).all(), c
        assert (np.diff(q[o, c]) >= 0).all(), c
        assert np.array_equal(np.diff(q[o, c]) == 0, np.diff(sim[o, c]) == 0), c
