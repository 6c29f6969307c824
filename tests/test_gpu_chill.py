"""Chill kernels on the GPU: bit for bit against the host build of chill_core.cuh (hourly temperatures, chill units,
valid counts; chill portions within the exp tolerance), the fused against the hourly-input path, and streamed
against device-resident inputs."""
import numpy as np
import pytest
import torch

import chill_host_build as H
from xclim_b200 import Field, TimeAxis, _lib, converters, device, indices
from xclim_b200.options import set_options

pytestmark = pytest.mark.gpu
K2C = 273.15
ALL = _lib.CHILL_PORTIONS | _lib.CHILL_UNITS


@pytest.fixture(scope="module", autouse=True)
def _release_hbm():
    """Hand the allocator's cached segments back after this module: the ~0.9 GB hourly float64 series it makes
    would otherwise stay reserved, and later modules that need most of the HBM (the full-size grid) could not get
    it."""
    yield
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _data(T, C, seed, ldx=None):
    rng = np.random.default_rng(seed)
    ldx = C if ldx is None else ldx
    lo = rng.uniform(-12, 14, (T, ldx)).astype(np.float32)
    hi = (lo + rng.uniform(0, 14, (T, ldx))).astype(np.float32)
    lo[rng.integers(0, T, 4), rng.integers(0, C, 4)] = np.nan        # NaN days
    lats = np.linspace(-90, 90, 37)[np.arange(C) % 37]                # polar rows included
    return lo, hi, lats


@pytest.mark.parametrize("C,ldx", [(1, 1), (37, 40), (129, 129), (4100, 4100)])
@pytest.mark.parametrize("cal,start", [("noleap", "2001-03-05"), ("360_day", "2001-01-01"), ("standard", "1999-08-20")])
@pytest.mark.parametrize("infill", [False, True])
def test_kernels_match_host_build(C, ldx, cal, start, infill):
    T = 3 * 365 + 40
    lo, hi, lats = _data(T, C, C + len(cal), ldx)
    ta = TimeAxis.daily(start, T, cal)
    lat_u, idx = np.unique(lats, return_inverse=True)
    idx = idx.astype(np.int32)
    w = converters.hourly_weights(ta, lat_u, infill)
    poff = ta.period_offsets("YS-JUL")                  # partial first and last periods
    mask = ta.select_mask(date_bounds=("09-01", "03-30"))
    lo_d, hi_d = torch.from_numpy(lo).cuda()[:, :C], torch.from_numpy(hi).cuda()[:, :C]
    w_d, idx_d = torch.from_numpy(w).cuda(), torch.from_numpy(idx).cuda()
    hr = device.hourly_temperature(lo_d, hi_d, w_d, idx_d).cpu().numpy()
    hr_h = H.hourly_temperature(lo, hi, w, idx, C=C)
    np.testing.assert_array_equal(hr, hr_h)
    hr_d = torch.from_numpy(hr).cuda()
    for pos in (False, True):
        what = ALL | (_lib.CHILL_POSITIVE_ONLY if pos else 0)
        for m in (None, mask):
            cp, cu, valid = (t.cpu().numpy() for t in device.chill_daily(lo_d, hi_d, w_d, idx_d, poff, m, (1.0, K2C),
                                                                         (1.0, 0.0), what, want_valid=True))
            cp2, cu2, valid2 = (t.cpu().numpy() for t in device.chill_hourly(hr_d, poff, m, (1.0, K2C), (1.0, 0.0),
                                                                             what, want_valid=True))
            cp_h, cu_h, valid_h = H.chill(poff, m, (1.0, K2C), (1.0, 0.0), what, tasmin=lo, tasmax=hi, weights=w,
                                          lat_index=idx, C=C)
            np.testing.assert_array_equal(cu, cu_h)
            np.testing.assert_array_equal(valid, valid_h)
            np.testing.assert_allclose(cp, cp_h, rtol=1e-11, atol=1e-12)
            for a, b in ((cp, cp2), (cu, cu2), (valid, valid2)):
                np.testing.assert_array_equal(a, b)


def test_hourly_float32_input():
    lo, hi, lats = _data(400, 64, 9)
    x = (np.repeat(lo, 24, 0)[:-5] + K2C).astype(np.float32)
    poff = np.array([0, 100, 400], np.int32)
    cp, cu, valid = (t.cpu().numpy() for t in device.chill_hourly(torch.from_numpy(x).cuda(), poff, None,
                                                                  (1.0, 0.0), (1.0, -K2C), ALL, want_valid=True))
    cp_h, cu_h, valid_h = H.chill(poff, None, (1.0, 0.0), (1.0, -K2C), ALL, hourly=x)
    np.testing.assert_array_equal(cu, cu_h)
    np.testing.assert_array_equal(valid, valid_h)
    np.testing.assert_allclose(cp, cp_h, rtol=1e-11, atol=1e-12)


def test_streamed_equals_device_resident():
    T, Y, X = 2 * 365, 6, 1440
    lo, hi, _ = _data(T, Y * X, 5)
    lats = np.linspace(-75, 75, Y)
    ta = TimeAxis.daily("2001-01-01", T, "noleap")

    def fields(on_dev):
        mk = (lambda v: torch.from_numpy(v.reshape(T, Y, X)).cuda()) if on_dev else (lambda v: v.reshape(T, Y, X))
        c = {"lat": lats}
        return (Field(mk(lo), ("time", "lat", "lon"), ta, c, {"units": "degC"}, "tasmin"),
                Field(mk(hi), ("time", "lat", "lon"), ta, c, {"units": "degC"}, "tasmax"))
    with set_options(stream_min_bytes=1 << 20, stream_slab_bytes=4 << 20):
        h = indices.make_hourly_temperature(*fields(False))
        a = indices.chill_portions(h, date_bounds=("09-01", "03-30"), freq="YS-JUL")
        b = indices.chill_units(h, positive_only=True)
    h2 = indices.make_hourly_temperature(*fields(True))
    a2 = indices.chill_portions(h2, date_bounds=("09-01", "03-30"), freq="YS-JUL")
    b2 = indices.chill_units(h2, positive_only=True)
    np.testing.assert_array_equal(np.asarray(a.values), np.asarray(a2.values.cpu() if hasattr(a2.values, "cpu")
                                                                   else a2.values))
    np.testing.assert_array_equal(np.asarray(b.values), np.asarray(b2.values.cpu() if hasattr(b2.values, "cpu")
                                                                   else b2.values))
