"""Potential evapotranspiration on the GPU: the kernels against the host build of the same device code
(tests/csrc/pet_host.cpp) on 1 to 4100 cells, an ldx > C view, three calendars and partial first and last
months, and the public functions end to end, streamed and not, against the oracle."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import pet_host_build as H  # noqa: E402
from oracle import pet_oracle as O  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]


def _series(T, C, rng, pad=0):
    tn = rng.uniform(-25, 25, (T, C)).astype(np.float32)
    tx = (tn + rng.uniform(-3, 15, (T, C))).astype(np.float32)
    tn[0, 0], tx[1 % T, C - 1] = np.nan, np.inf
    return {"tasmin": tn, "tasmax": tx, "tas": ((tn + tx) / 2).astype(np.float32),
            "hurs": rng.uniform(0.05, 1, (T, C)).astype(np.float32),
            "rsds": rng.uniform(0, 400, (T, C)).astype(np.float32), "rsus": rng.uniform(0, 80, (T, C)).astype(np.float32),
            "rlds": rng.uniform(200, 400, (T, C)).astype(np.float32),
            "rlus": rng.uniform(200, 450, (T, C)).astype(np.float32),
            "sfcWind": rng.uniform(0, 15, (T, C)).astype(np.float32),
            "pr": rng.uniform(0, 5e-4, (T, C)).astype(np.float32)}


def _dev(x, pad):
    import torch
    T, C = x.shape
    buf = torch.full((T, C + pad), 7.0, dtype=torch.float32, device="cuda")
    buf[:, :C] = torch.from_numpy(x).cuda()
    return buf[:, :C]


NEEDS = {"BR65": ("tasmin", "tasmax"), "HG85": ("tasmin", "tasmax", "tas"), "MB05": ("tasmin", "tasmax"),
         "allen98": ("tasmin", "tasmax", "hurs", "rsds", "rsus", "rlds", "rlus", "sfcWind")}


@pytest.mark.parametrize("method", list(NEEDS))
@pytest.mark.parametrize("C,pad,wb", [(1, 0, False), (33, 3, True), (4100, 0, True), (257, 31, False)])
def test_daily_kernel_matches_host_build(method, C, pad, wb):
    import torch
    from xclim_b200 import TimeAxis, _lib, converters, device
    rng = np.random.default_rng(C)
    ta = TimeAxis.daily("2000-02-20", 50, "standard")            # leap day, partial months
    s = _series(len(ta), C, rng)
    lats = rng.choice(np.array([-90.0, -70.0, -12.0, 0.0, 45.0, 66.6, 89.0]), C)
    lat_u, idx = np.unique(lats, return_inverse=True)
    table = None if method == "allen98" else converters._daily_table(method, ta, lat_u)
    names = NEEDS[method] + (("pr",) if wb else ())
    host_in = [s[n] if n in names else None for n in _lib.PET_INPUTS]
    P = H.params(method, wb)
    ref = H.daily(host_in, table, None if table is None else idx, P)
    dev_in = [None if x is None else _dev(x, pad) for x in host_in]
    got = device.pet_daily(dev_in, None if table is None else torch.from_numpy(table).cuda(),
                           None if table is None else torch.from_numpy(idx.astype(np.int32)).cuda(), P)
    got = got.cpu().numpy()
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    if method == "allen98":      # the device exp / log
        f = np.isfinite(ref)
        np.testing.assert_array_max_ulp(got[f], ref[f], maxulp=1)
    else:
        np.testing.assert_array_equal(got, ref)


@pytest.mark.parametrize("method", ["TW48", "DA02"])
@pytest.mark.parametrize("calendar,start,n,C,pad", [("standard", "1999-11-17", 500, 33, 2), ("360_day", "2001-02-03", 400, 1, 0),
                                                    ("noleap", "2003-12-31", 70, 4100, 0)])
def test_monthly_kernel_matches_host_build(method, calendar, start, n, C, pad):
    import torch
    from xclim_b200 import TimeAxis, _lib, converters, device
    rng = np.random.default_rng(n)
    ta = TimeAxis.daily(start, n, calendar)
    s = _series(len(ta), C, rng)
    s["pr"] = (s["pr"] * np.float32(1e5)).astype(np.float32)
    lats = rng.choice(np.array([-80.0, 0.0, 45.0, 70.0]), C)
    lat_u, idx = np.unique(lats, return_inverse=True)
    moff, yoff, ym, mdays = converters._months(ta)
    table = converters._monthly_table(method, ta, ym, lat_u)
    names = ("tasmin", "tasmax", "pr") if method == "DA02" else ("tas", "pr")
    host_in = [s[n_] if n_ in names else None for n_ in _lib.PET_INPUTS]
    P = H.params(method, method == "TW48")
    ref = H.monthly(host_in, moff, yoff, mdays, table, idx, P)
    got = device.pet_monthly([None if x is None else _dev(x, pad) for x in host_in], moff, yoff, mdays,
                             torch.from_numpy(table).cuda(), torch.from_numpy(idx.astype(np.int32)).cuda(), P)
    got = got.cpu().numpy()
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    f = np.isfinite(ref)
    np.testing.assert_array_max_ulp(got[f], ref[f], maxulp=1)


@pytest.mark.parametrize("stream", [False, True])
def test_water_budget_end_to_end(stream):
    import torch
    from xclim_b200 import Field, TimeAxis, indices, set_options
    rng = np.random.default_rng(11)
    ta = TimeAxis.daily("2001-01-01", 3 * 365, "noleap")
    T, nl, nx = len(ta), 6, 40
    tn = rng.uniform(260, 290, (T, nl, nx)).astype(np.float32)
    tx = (tn + rng.uniform(1, 12, (T, nl, nx))).astype(np.float32)
    pr = rng.gamma(0.8, 3.0, (T, nl, nx)).astype(np.float32)
    lat = np.linspace(-60, 60, nl)

    def f(v, u):
        return Field(v, ("time", "lat", "lon"), ta, {"lat": lat}, {"units": u})

    opts = {"stream_min_bytes": 1, "stream_slab_bytes": T * nx * 4 * 2} if stream else {}
    with set_options(**opts):
        wb = indices.water_budget(f(pr, "mm/d"), tasmin=f(tn, "K"), tasmax=f(tx, "K"), method="BR65")
    table = O.radiation_table(ta.year, ta.doy, "noleap", lat) * (1 / 41840.0)
    conv = lambda x: (x * np.float32(1.8) + np.float32(-459.67)).astype(np.float32)  # noqa: E731
    prk = (pr * np.float32(1 / 86400)).astype(np.float32)
    ref = np.float32(O.daily_rate(O.daily_pet("BR65", table[:, :, None], tasmin=conv(tn), tasmax=conv(tx)), prk))
    got = np.asarray(wb.values)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-12)
    # device-resident inputs stay on the device
    with set_options(device_outputs=True):
        d = indices.water_budget(f(torch.from_numpy(pr).cuda(), "mm/d"), tasmin=f(torch.from_numpy(tn).cuda(), "K"),
                                 tasmax=f(torch.from_numpy(tx).cuda(), "K"), method="BR65")
        assert d.values.is_cuda
        np.testing.assert_array_equal(d.values.cpu().numpy(), got)
        spei = indices.standardized_precipitation_evapotranspiration_index(d, freq="MS", window=1, dist="gamma",
                                                                           method="APP", fitkwargs={"floc": -1e-3})
        out = spei.values.cpu().numpy()
    assert out.shape == (36, nl, nx) and spei.dims == ("time", "lat", "lon")
    # the oracle composition: the monthly means of the oracle's water budget, then the oracle's fit and transform,
    # compared with the rule of test_gpu_stdindex.py (the monthly means of the kernel within one float32 ulp, the
    # index within 1e-13 after weighting by the normal density)
    import scipy.stats as st
    from oracle import stdindex_oracle as SO
    from oracle import xclim_oracle as XO
    from xclim_b200 import stats
    poff = ta.period_offsets("MS")
    y_o = XO.resample_reduce(ref.reshape(T, -1).astype(np.float64), poff, "mean").astype(np.float32)
    series, _, _, _ = stats._preprocess(d, "MS", 1, {})
    y = series.y.cpu().numpy()
    np.testing.assert_array_max_ulp(y, y_o, maxulp=1)
    gid = np.asarray(series.group)
    np.testing.assert_array_equal(gid, ta.month[poff[:-1]] - 1)
    po, _, _ = SO.fit_groups(y, gid, 12, slice(None), "gamma", "APP", False, -1e-3)
    sio = SO.transform(y, gid, po, "gamma").reshape(out.shape)
    good = ~np.isnan(sio)
    assert good.mean() > 0.9
    np.testing.assert_array_equal(np.isnan(out), ~good)
    assert np.all(np.abs(out - sio)[good] * st.norm.pdf(sio[good]) <= 1e-13)
