"""Spatial analogues without a GPU: the oracle against the reference's goldens and its tests' known answers, the
host build of analog_core.cuh against the oracle, the host layer of xclim_b200.analog over an oracle-backed
stand-in of the kernel, and the C argument checks."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import scipy.stats as st
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import analog_host_build as H  # noqa: E402
import mini_xarray as mx  # noqa: E402
from oracle import analog_oracle as O  # noqa: E402
from xclim_b200 import Field, analog, set_options  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_analog.npz")
#: golden column -> (metric, oracle kwargs, kernel param)
COLUMNS = {"seuclidean": ("seuclidean", {}, 0.0), "nearest_neighbor": ("nearest_neighbor", {}, 0.0),
           "zech_aslan": ("zech_aslan", {}, 1e-12), "szekely_rizzo": ("szekely_rizzo", {}, 1.0),
           "szekely_rizzo_raw": ("szekely_rizzo", {"standardize": False}, 0.0),
           "kolmogorov_smirnov": ("kolmogorov_smirnov", {}, 0.0), "kldiv": ("kldiv", {}, 1.0),
           "kldiv_k3": ("kldiv", {"k": 3}, 3.0), "mahalanobis": ("mahalanobis", {}, 0.0)}
EXACT = ("nearest_neighbor", "kolmogorov_smirnov")


def _golden():
    g = np.load(GOLDEN)
    cases = [(str(nm), g[f"x_{i}"], g[f"y_{i}"]) for i, nm in enumerate(g["names"])]
    return g, cases


def _oracle(col, x, y):
    meth, kw, _ = COLUMNS[col]
    try:
        return O.metric(meth, x, y, **kw), ""
    except Exception as e:  # noqa: BLE001 - compared with the recorded exception
        return np.nan, f"{type(e).__name__}: {e}"


def _nn_margin(x, y):
    """Smallest relative gap between the nearest and second-nearest squared distances over the pooled points."""
    _, sx = O._seq_stats(np.asarray(x, float))
    _, sy = O._seq_stats(np.asarray(y, float))
    z = np.vstack([x, y]) / np.sqrt(sx * sy)
    d = O._pair_dists(z, z, squared=True)
    np.fill_diagonal(d, np.inf)
    s = np.sort(d, axis=1)
    with np.errstate(invalid="ignore"):
        return float(np.min(np.nan_to_num((s[:, 1] - s[:, 0]) / s[:, 1], nan=0.0)))   # 0 / 0: a tie at 0


# ------------------------------------------------------------------------------------ oracle vs reference
def test_golden_metric_names_and_order():
    g, _ = _golden()
    assert list(g["metrics"]) == O.METRICS == analog.metrics


def test_oracle_matches_reference_goldens():
    g, cases = _golden()
    cols = list(g["columns"])
    n_nn = 0
    for i, (name, x, y) in enumerate(cases):
        f32 = x.dtype == np.float32
        for j, col in enumerate(cols):
            ref, err = g["values"][i, j], str(g["errors"][i, j])
            got, gerr = _oracle(col, x, y)
            if col == "nearest_neighbor" and not err and np.isfinite(ref):
                # ties are broken by a stated rule here, by cKDTree's traversal in the reference: compare only
                # where every neighbour is clear of the float32 standardization error
                if _nn_margin(x, y) < 1e-4:
                    continue
                n_nn += 1
            assert gerr == err, (name, col)
            if err:
                continue
            if not np.isfinite(ref):
                assert (np.isnan(ref) and np.isnan(got)) or ref == got, (name, col, ref, got)
            elif col in EXACT:
                assert got == ref, (name, col)
            else:
                np.testing.assert_allclose(got, ref, rtol=1e-5 if f32 else 1e-12, atol=0, err_msg=f"{name} {col}")
    assert n_nn >= 30


def test_reference_raises_where_stated():
    g, cases = _golden()
    cols = list(g["columns"])
    err = {(n, c): str(g["errors"][i, j]) for i, (n, _, _) in enumerate(cases) for j, c in enumerate(cols)}
    kd = "ValueError: " + O.MSG_KDTREE
    for tag in ("posinf", "neginf"):
        for where in ("target", "cand"):
            case = f"{tag}_{where}_float32"
            assert err[(case, "seuclidean")] == "ValueError: " + O.MSG_CHKFINITE
            assert err[(case, "nearest_neighbor")] == err[(case, "kldiv")] == kd
            for c in ("zech_aslan", "szekely_rizzo", "kolmogorov_smirnov", "mahalanobis"):
                assert err[(case, c)] == "", (case, c)       # mahalanobis: IEEE inf / NaN, no raise
    assert err[("const_cand_float64", "nearest_neighbor")] == kd
    assert err[("const_target_float64", "seuclidean")] == "ValueError: " + O.MSG_CHKFINITE
    assert err[("posinf_small_target_float64", "kldiv")] == ""     # n < 5: NaN before the finiteness check
    assert err[("normal_n5_m6_d10_float64", "kldiv")] == ""                 # d = 10 is allowed


def test_oracle_known_answers():
    z = 1.0 * (np.arange(30) + 1) / 30 - 0.5
    x = np.vstack([z * 2 + 30, z * 3 + 40, z]).T
    y = np.vstack([z * 2.2 + 31, z[::-1] * 2.8 + 38, z * 1.1]).T
    np.testing.assert_almost_equal(O.metric("seuclidean", x, y), 2.8463, 4)
    np.testing.assert_almost_equal(O.metric("nearest_neighbor", x, y), 1, 4)
    np.testing.assert_almost_equal(O.metric("zech_aslan", x, y), 0.77802, 4)
    np.testing.assert_almost_equal(O.metric("kolmogorov_smirnov", x, y), 0.96667, 4)


def _exact_randn(rng, mean, std, shape):
    r = rng.standard_normal(shape)
    r1 = r / r.std(0, ddof=1) * np.array(std)
    return r1 - r1.mean(0) + np.array(mean)


def test_oracle_and_host_build_reference_checks():
    """The reference tests' exact-randn, ks_2samp, nearest-neighbour and analytic-KL checks at their decimals."""
    rng = np.random.default_rng(42)
    for std in (1, 2):
        x = _exact_randn(rng, 0, 1, (25, 2))
        y = _exact_randn(rng, [1, 2], std, (30, 2))
        np.testing.assert_almost_equal(O.metric("seuclidean", x, y), np.hypot(1, 2), 2)
    a, b = rng.standard_normal(50) + 1, rng.standard_normal(50)
    np.testing.assert_almost_equal(O.metric("kolmogorov_smirnov", a, b), st.ks_2samp(a, b)[0], 3)
    x, y = rng.standard_normal((200, 2)), rng.standard_normal((200, 2))
    np.testing.assert_almost_equal(O.metric("nearest_neighbor", x + 0.001, x), 0, 2)
    np.testing.assert_almost_equal(O.metric("nearest_neighbor", x, y), 0.5, 1)
    np.testing.assert_almost_equal(O.metric("nearest_neighbor", x + 10, y), 1, 2)
    assert O.metric("zech_aslan", x + 0.001, x) < 0
    # analytic KL divergence of N(2, 1) from N(2.6, 1.4), on 10000 points through the host build
    p, q = st.norm(2, 1), st.norm(2.6, 1.4)
    ra = np.log(1.4) + (1 + 0.6 ** 2) / (2 * 1.4 ** 2) - 0.5
    xs, ys = p.rvs(10000, random_state=rng), q.rvs(10000, random_state=rng)
    got, status = H.analog(xs[None, :, None], ys[None, :, None], "kldiv", 1.0)
    assert status == 0
    np.testing.assert_almost_equal(got[0, 0], ra, 1)


# ------------------------------------------------------------------------------------ host build vs oracle
def test_host_build_matches_oracle_on_every_golden_case():
    _, cases = _golden()
    for name, x, y in cases:
        for col, (meth, kw, param) in COLUMNS.items():
            want, werr = _oracle(col, x, y)
            if werr.startswith(("LinAlgError", "ValueError: Too many")):
                continue                     # raised by the host layer before the kernel
            cst = O.target_consts(x, meth)
            got, status = H.analog(x[None], y[None], meth, param, None if cst is None else np.asarray(cst)[None])
            gerr = {0: "", analog._lib.AN_STATUS_NOT_FINITE: "ValueError: " + O.MSG_KDTREE,
                    analog._lib.AN_STATUS_CHKFINITE: "ValueError: " + O.MSG_CHKFINITE}[status]
            assert gerr == werr, (name, col)
            if werr:
                continue
            got = got[0, 0]
            if col in EXACT or not np.isfinite(want):
                assert got == want or (np.isnan(got) and np.isnan(want)), (name, col, got, want)
            else:
                np.testing.assert_allclose(got, want, rtol=1e-12, atol=0, err_msg=f"{name} {col}")


# ------------------------------------------------------------------------------------ host layer
def _fake_analog(target, cand, method_code, param, consts):
    """Oracle-backed stand-in for device.analog: targets (K, n, d), candidates (m, d, C)."""
    meth = {v: k for k, v in analog._lib.AN_METHODS.items()}[method_code]
    t, y = target.cpu().numpy(), cand.cpu().numpy()
    K, n, d = t.shape
    out = np.empty((K, y.shape[2]))
    status = 0
    for k in range(K):
        for c in range(y.shape[2]):
            kw = {"seuclidean": {}, "mahalanobis": {}, "zech_aslan": {"dmin": param},
                  "szekely_rizzo": {"standardize": bool(param)}, "kldiv": {"k": int(param)}}.get(meth, {})
            if consts is not None and meth == "mahalanobis":
                kw["VI"] = consts[k].cpu().numpy().reshape(d, d)
            if consts is not None and meth == "seuclidean":
                kw["V"] = consts[k].cpu().numpy()
            try:
                out[k, c] = O.metric(meth, t[k], y[:, :, c], **kw)
            except ValueError as e:
                status |= analog._lib.AN_STATUS_CHKFINITE if str(e) == O.MSG_CHKFINITE else \
                    analog._lib.AN_STATUS_NOT_FINITE
                out[k, c] = np.nan
    return torch.from_numpy(out), status


@pytest.fixture
def fake(monkeypatch):
    from xclim_b200 import device
    monkeypatch.setattr(device, "analog", _fake_analog)
    monkeypatch.setattr(analog, "_DEVICE", "cpu")


def _grid(rng, T, lat, lon, names=("a", "b", "c"), order=("time", "lat", "lon"), field=True):
    out = {}
    for i, v in enumerate(names):
        a = rng.normal(10 * (i + 1), 1 + i, (T, lat, lon)).astype(np.float32)
        a = np.transpose(a, [("time", "lat", "lon").index(d) for d in order])
        out[v] = Field(a, order, None, {}, {}, v) if field else mx.DataArray(a, dims=order, name=v)
    return out


def _expected(target, cand, method, dist_dim="time", **kw):
    """The oracle cell by cell over the stacked inputs."""
    tv, trest = analog._stack(target, dist_dim, "target")
    cv, crest = analog._stack(cand, dist_dim, "candidates")
    tv, cv = np.asarray(tv, np.float64), np.asarray(cv, np.float64)
    out = np.empty(tv.shape[:-2] + cv.shape[:-2])
    for ti in np.ndindex(tv.shape[:-2]):
        for ci in np.ndindex(cv.shape[:-2]):
            out[ti + ci] = O.metric(method, tv[ti], cv[ci], **kw)
    return out, trest + crest


@pytest.mark.parametrize("method", ["seuclidean", "nearest_neighbor", "zech_aslan", "szekely_rizzo",
                                    "kolmogorov_smirnov", "kldiv", "mahalanobis"])
def test_host_layer_dims_sites_and_lengths(fake, method):
    rng = np.random.default_rng(3)
    cand = _grid(rng, 31, 3, 4, order=("lat", "time", "lon"))
    target = {k: Field(v.values[:2, :20, 1].T, ("time", "site"), None, {}, {}, k) for k, v in cand.items()}
    out = analog.spatial_analogs(target, cand, method=method)
    want, dims = _expected(target, cand, method)
    assert out.dims == dims == ("site", "lat", "lon") and out.name == "dissimilarity"
    assert out.values.dtype == np.float64 and out.values.shape == (2, 3, 4)
    np.testing.assert_allclose(out.values, want, rtol=1e-12)
    assert out.attrs == {"long_name": f"Dissimilarity between target and candidates, using metric {method}.",
                         "indices": "a,b,c", "metric": method}


def test_host_layer_mini_xarray_and_sample_dim(fake, monkeypatch):
    mx.install(monkeypatch)
    rng = np.random.default_rng(4)
    cand = _grid(rng, 12, 2, 3, names=("tg", "fd"), order=("lon", "lat", "time"), field=False)
    cand = {k: mx.DataArray(v.values, dims=("lon", "lat", "sample"), name=k) for k, v in cand.items()}
    target = {k: mx.DataArray(v.values[1, 0, :9], dims=("sample",), name=k) for k, v in cand.items()}
    out = analog.spatial_analogs(target, cand, dist_dim="sample", method="zech_aslan", dmin=1e-6)
    assert isinstance(out, mx.DataArray) and out.dims == ("lon", "lat")
    want, _ = _expected(target, cand, "zech_aslan", dist_dim="sample", dmin=1e-6)
    np.testing.assert_allclose(out.values, want, rtol=1e-12)


def test_host_layer_device_outputs(fake):
    rng = np.random.default_rng(5)
    cand = _grid(rng, 10, 2, 2)
    target = {k: Field(v.values[:, 0, 0], ("time",), None, {}, {}, k) for k, v in cand.items()}
    with set_options(device_outputs=True):
        out = analog.spatial_analogs(target, cand, method="seuclidean")
    assert isinstance(out.values, torch.Tensor)


def test_host_layer_errors(fake):
    rng = np.random.default_rng(6)
    cand = _grid(rng, 10, 2, 2)
    target = {k: Field(v.values[:, 0, 0], ("time",), None, {}, {}, k) for k, v in cand.items()}
    with pytest.raises(ValueError, match="Method `KonMari` is not implemented. Available methods are: "
                                         "seuclidean,nearest_neighbor,zech_aslan,szekely_rizzo,friedman_rafsky,"
                                         "kolmogorov_smirnov,kldiv,mahalanobis."):
        analog.spatial_analogs(target, cand, method="KonMari")
    with pytest.raises(NotImplementedError, match="kneighbors_graph"):
        analog.spatial_analogs(target, cand, method="friedman_rafsky")
    with pytest.raises(NotImplementedError, match="sequence of k"):
        analog.spatial_analogs(target, cand, method="kldiv", k=[1, 2])
    with pytest.raises(NotImplementedError, match="one dimension name"):
        analog.spatial_analogs(target, cand, dist_dim=["time"], method="kldiv")
    with pytest.raises(ValueError, match="join='exact'"):
        analog.spatial_analogs({k: target[k] for k in ("b", "a", "c")}, cand, method="seuclidean")
    with pytest.raises(TypeError, match="unexpected keyword argument 'k'"):
        analog.spatial_analogs(target, cand, method="seuclidean", k=2)
    with pytest.raises(AttributeError, match="VI not a matrix"):
        analog.spatial_analogs(target, cand, method="mahalanobis", VI=[[1.0]])
    one = {"a": target["a"]}
    with pytest.raises(np.linalg.LinAlgError):
        analog.spatial_analogs(one, {"a": cand["a"]}, method="mahalanobis")
    wide = _grid(rng, 10, 1, 2, names=tuple("abcdefghijk"))
    wt = {k: Field(v.values[:, 0, 0], ("time",), None, {}, {}, k) for k, v in wide.items()}
    with pytest.raises(ValueError, match=r"Too many dimensions: 11\."):
        analog.spatial_analogs(wt, wide, method="kldiv")
    bad = dict(cand)
    bad["b"] = Field(cand["b"].values.copy(), cand["b"].dims, None, {}, {}, "b")
    bad["b"].values[3, 1, 0] = np.inf
    with pytest.raises(ValueError, match="array must not contain infs or NaNs"):
        analog.spatial_analogs(target, bad, method="seuclidean")
    for meth in ("nearest_neighbor", "kldiv"):
        with pytest.raises(ValueError, match="data must be finite, check for nan or inf values"):
            analog.spatial_analogs(target, bad, method=meth)
    out = analog.spatial_analogs(target, bad, method="zech_aslan")         # IEEE, no raise
    assert np.isnan(out.values[1, 0]) and np.isfinite(out.values[0, 0])


# ------------------------------------------------------------------------------------ C argument checks
def test_c_argument_checks():
    from xclim_b200 import _build, _lib
    if not os.path.exists(_build.LIB_PATH):
        _build.build()
    lib = _lib.load()
    buf = (C.c_double * 4096)()
    p = C.cast(buf, C.c_void_p)

    def call(t=p, n=30, K=1, y=p, m=30, Cc=64, ldc=64, d=3, method=2, param=1e-12, cst=None, out=p, st=p):
        return lib.xc_analog_f32(t, n, K, y, m, Cc, ldc, d, method, param, cst, out, st, None)

    assert call(t=None) == -1 and b"null pointer" in lib.xc_last_error()
    assert call(method=7) == -1 and b"unknown analogue method" in lib.xc_last_error()
    for kw in ({"n": 0}, {"m": 0}, {"K": 0}, {"K": 65536}, {"Cc": 0}, {"ldc": 63}):
        assert call(**kw) == -1 and b"bad shape" in lib.xc_last_error(), kw
    for d in (0, 17):
        assert call(d=d) == -1 and b"number of indicators" in lib.xc_last_error()
    for meth in (0, 6):
        assert call(method=meth) == -1 and b"per-target constants" in lib.xc_last_error()
    assert call(method=5, d=11) == -1 and b"Too many dimensions: 11." in lib.xc_last_error()
    for k in (0.0, 17.0, 1.5):
        assert call(method=5, param=k) == -1 and b"integer k" in lib.xc_last_error()
    assert call(n=2000, m=2000, d=16) == -1 and b"too large" in lib.xc_last_error()
