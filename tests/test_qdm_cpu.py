"""Quantile delta mapping without a GPU: the oracle (oracle/qdm_oracle.py: qdm_rank, qdm_adjust) against a literal
per-cell restatement and known answers, the host wrapper sdba.QuantileDeltaMapping over oracle-backed device functions, and
the argument validation of xc_qdm_adjust_f32 through the real library."""
import ctypes as C

import numpy as np
import pytest
import torch

import fake_device
from oracle import qdm_oracle as Q
from oracle import xclim_oracle as O
from xb_helpers import make_field


def literal_rank(col):
    """sim_q of one series, element by element: r = #{valid < x} + (#{valid == x} + 1) / 2, p = r / n, then
    (mx * (p - mn)) / (mx - mn)."""
    valid = [float(v) for v in col if v == v]
    n = len(valid)
    p = [np.nan if v != v else (sum(w < v for w in valid) + (sum(w == v for w in valid) + 1) / 2) / n for v in col]
    ps = [x for x in p if x == x]
    if not ps:
        return np.array(p)
    mn, mx = min(ps), max(ps)
    with np.errstate(all="ignore"):
        return np.array([np.nan if x != x else (np.float64(mx) * (x - mn)) / np.float64(mx - mn) for x in p])


def test_rank_known_answers():
    inc = np.arange(7, dtype=np.float32)[:, None]
    got = Q.qdm_rank(inc)[:, 0]
    assert got.dtype == np.float64 and got[0] == 0.0 and got[-1] == 1.0
    np.testing.assert_allclose(got, np.linspace(0, 1, 7), rtol=0, atol=1e-15)
    # ties get the average rank: ranks 1, 2.5, 2.5, 4 -> p = r / 4 -> rescaled by (mx * (p - mn)) / (mx - mn)
    tie = np.array([1.0, 2.0, 2.0, 3.0], np.float32)[:, None]
    p = np.array([1, 2.5, 2.5, 4]) / 4
    np.testing.assert_array_equal(Q.qdm_rank(tie)[:, 0], (1.0 * (p - 0.25)) / 0.75)
    # -0.0 and +0.0 are one tie group; NaN stays NaN; +-inf are ordinary extremes
    z = np.array([0.0, -0.0, np.nan, np.inf, -np.inf], np.float32)[:, None]
    q = Q.qdm_rank(z)[:, 0]
    assert q[0] == q[1] and np.isnan(q[2]) and q[3] == 1.0 and q[4] == 0.0
    # a constant cell, a one-valid cell and an all-NaN cell are NaN throughout
    deg = np.full((5, 3), np.nan, np.float32)
    deg[:, 0] = 2.5
    deg[3, 1] = 1.0
    assert np.isnan(Q.qdm_rank(deg)).all()


def test_rank_matches_literal_restatement():
    rng = np.random.default_rng(11)
    x = np.round(rng.gamma(0.5, 3.0, (60, 6)) * 2).astype(np.float32) / 2   # many ties
    x[rng.random(x.shape) < 0.4] = 0.0
    x[rng.random(x.shape) < 0.05] = np.nan
    x[:5, 2] = -0.0
    x[7, 3], x[9, 3] = np.inf, -np.inf
    got = Q.qdm_rank(x)
    for c in range(x.shape[1]):
        np.testing.assert_array_equal(got[:, c], literal_rank(x[:, c]), err_msg=str(c))


def test_adjust_factor_known_answers():
    """af linear in the nodes: the linear factor is that line at sim_q, constant beyond the end nodes; nearest picks
    the closest node, ties to the lower one; NaN af entries are dropped; scen in float32."""
    nq = 4
    nodes = O.eqm_nodes(nq).astype(np.float32)                   # 0.125, 0.375, 0.625, 0.875
    af = (10 * nodes).astype(np.float32)[:, None]
    sim = np.arange(9, dtype=np.float32)[:, None]                # sim_q = 0, 1/8, ..., 1
    scen, q = Q.qdm_adjust(sim, af, "+", "linear")
    np.testing.assert_allclose(q[:, 0], np.arange(9) / 8, rtol=0, atol=1e-15)
    exp = np.clip(10 * np.arange(9) / 8, 1.25, 8.75)
    np.testing.assert_allclose(scen[:, 0] - sim[:, 0], exp, rtol=1e-6)
    assert scen.dtype == np.float32
    scen_n, _ = Q.qdm_adjust(sim, af, "*", "nearest", sim_q=(np.arange(9) / 8)[:, None])
    # q = 2/8 lies exactly between the nodes 1/8 and 3/8: the lower one
    np.testing.assert_allclose(scen_n[:, 0] / np.where(sim[:, 0] == 0, 1, sim[:, 0]),
                               np.where(sim[:, 0] == 0, 0, [1.25, 1.25, 1.25, 3.75, 3.75, 6.25, 6.25, 8.75, 8.75]),
                               rtol=1e-6)
    af_nan = af.copy()
    af_nan[1:3] = np.nan                                         # only the end nodes remain
    scen_l, _ = Q.qdm_adjust(sim, af_nan, "+", "linear")
    np.testing.assert_allclose(scen_l[:, 0] - sim[:, 0],
                               1.25 + (np.clip(np.arange(9) / 8, 0.125, 0.875) - 0.125) * 10, rtol=1e-6)


# ---- the host wrapper over oracle-backed device functions
def fake_qdm_adjust(sim2d, af, nodes, kind_code, interp_code, want_sim_q=False, workspace_bytes=None):
    np.testing.assert_array_equal(np.asarray(nodes), O.eqm_nodes(af.shape[0]).astype(np.float32))
    scen, q = Q.qdm_adjust(sim2d.numpy(), af.numpy(), "+" if kind_code == 0 else "*",
                           "linear" if interp_code == 1 else "nearest")
    return torch.from_numpy(np.ascontiguousarray(scen)), (torch.from_numpy(q) if want_sim_q else None)


@pytest.fixture
def host(monkeypatch):
    fake_device.install(monkeypatch)
    from xclim_b200 import device
    monkeypatch.setattr(device, "qdm_adjust", fake_qdm_adjust)


def _series(seed, T=730, shape=(2, 3)):
    rng = np.random.default_rng(seed)
    ref = (285 + 6 * rng.standard_normal((T,) + shape)).astype(np.float32)
    hist = (286.5 + 7 * rng.standard_normal((T,) + shape)).astype(np.float32)
    sim = (288.5 + 7 * rng.standard_normal((T + 365,) + shape) + np.linspace(0, 3, T + 365)[:, None, None])
    return ref, hist, sim.astype(np.float32)


def test_qdm_host_wrapper(host):
    import xclim_b200
    from xclim_b200 import sdba
    ref, hist, sim = _series(9)
    f = lambda a: make_field(a, "1981-01-01", calendar="noleap", units="K")  # noqa: E731
    qdm = sdba.QuantileDeltaMapping.train(f(ref), f(hist), nquantiles=15, kind="+", group="time")
    eqm = sdba.EmpiricalQuantileMapping.train(f(ref), f(hist), nquantiles=15, kind="+", group="time")
    assert isinstance(qdm, sdba.EmpiricalQuantileMapping)
    for k in ("af", "hist_q"):                                   # train is EQM's
        np.testing.assert_array_equal(qdm.ds[k].values, eqm.ds[k].values)
        assert qdm.ds[k].dims == eqm.ds[k].dims
    scen = qdm.adjust(f(sim), interp="linear")                   # sim longer than the training series
    exp, q = Q.qdm_adjust(sim, qdm.ds["af"].values, "+", "linear")
    np.testing.assert_array_equal(scen.values, exp)
    assert scen.values.dtype == np.float32 and scen.values.shape == sim.shape
    assert scen.attrs["units"] == "K" and scen.dims == f(sim).dims
    with xclim_b200.set_options(sdba_extra_output=True):
        out = qdm.adjust(f(sim), interp="nearest")
    assert set(out) == {"scen", "sim_q"}
    assert out["sim_q"].values.dtype == np.float64 and out["sim_q"].values.shape == sim.shape
    np.testing.assert_array_equal(out["sim_q"].values, q)
    np.testing.assert_array_equal(out["scen"].values, Q.qdm_adjust(sim, qdm.ds["af"].values, "+", "nearest")[0])
    assert out["sim_q"].dims == scen.dims
    assert not isinstance(qdm.adjust(f(sim)), dict)               # the option is back to False
    # the same errors as EQM's adjust
    with pytest.raises(NotImplementedError):
        qdm.adjust(f(sim), interp="cubic")
    with pytest.raises(NotImplementedError):
        qdm.adjust(f(sim), extrapolation="nan")
    with pytest.raises(NotImplementedError):
        qdm.adjust(f(sim), adapt_freq_thresh="1 mm/d")
    with pytest.raises(ValueError):
        qdm.adjust(f(sim[:, :1]))
    with pytest.raises(NotImplementedError):
        sdba.QuantileDeltaMapping.train(f(ref), f(hist), group="time.month")
    with pytest.raises(ValueError):
        sdba.QuantileDeltaMapping.train(f(ref), f(hist), kind="-")
    with pytest.raises(ValueError, match="valid options"):
        xclim_b200.set_options(sdba_extra_outputs=True)


def test_eqm_adjust_unchanged_by_the_qdm_option(host):
    import xclim_b200
    from xclim_b200 import sdba
    ref, hist, sim = _series(10)
    f = lambda a: make_field(a, "1981-01-01", calendar="noleap", units="K")  # noqa: E731
    eqm = sdba.EmpiricalQuantileMapping.train(f(ref), f(hist), nquantiles=10, kind="*", group="time")
    plain = eqm.adjust(f(sim), interp="linear").values
    with xclim_b200.set_options(sdba_extra_output=True):
        again = eqm.adjust(f(sim), interp="linear")
    assert not isinstance(again, dict)
    np.testing.assert_array_equal(again.values, plain)


# ---- argument validation of the C entry point (host side, no device work)
@pytest.fixture(scope="module")
def lib():
    import os

    from xclim_b200 import _build, _lib
    if not os.path.exists(_build.LIB_PATH):
        _build.build()
    return _lib.load()


def test_qdm_argument_validation(lib):
    INVALID, UNSUPPORTED = -1, -2
    buf = (C.c_float * 16)()
    p = C.cast(buf, C.c_void_p)
    ws_min = lib.xc_qdm_adjust_workspace_bytes(4, 32)
    assert ws_min == 32 * (6 * 4 + 16) + 256
    assert lib.xc_qdm_adjust_workspace_bytes(10950, 259200) == 259200 * (6 * 10950 + 16) + 256
    assert lib.xc_qdm_adjust_workspace_bytes(4, 33) == lib.xc_qdm_adjust_workspace_bytes(4, 64)

    def call(sim=p, T=4, Cn=4, ldx=4, af=p, nodes=p, nq=20, kind=0, interp=1, scen=p, q=None, ws=p, wsb=ws_min):
        return lib.xc_qdm_adjust_f32(sim, T, Cn, ldx, af, nodes, nq, kind, interp, scen, q, ws, wsb, None)

    for kw in ({"sim": None}, {"af": None}, {"nodes": None}, {"scen": None}, {"ws": None}):
        assert call(**kw) == INVALID and b"null pointer" in lib.xc_last_error(), kw
    for kw in ({"T": 0}, {"Cn": 0}, {"ldx": 3}):
        assert call(**kw) == INVALID and b"shape" in lib.xc_last_error(), kw
    for nq in (1, 201):
        assert call(nq=nq) == INVALID and b"[2, 200]" in lib.xc_last_error()
    assert call(kind=2) == INVALID and b"kind" in lib.xc_last_error()
    assert call(interp=2) == INVALID and b"interp" in lib.xc_last_error()
    assert call(wsb=ws_min - 1) == INVALID and b"workspace too small" in lib.xc_last_error()
    assert call(T=32769, wsb=1 << 40) == UNSUPPORTED and b"32768" in lib.xc_last_error()
