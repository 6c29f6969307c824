"""Potential evapotranspiration and the water budget without a GPU: the host solar tables against the oracle's
day-by-day helpers, the host build of pet_core.cuh against the oracle's float64 mode on hostile inputs, the host
layer of xclim_b200.converters over a stand-in of the kernels built from the same host build (the reference tests'
known answers, aliases, units, the lat forms, MS labels, errors), and the C argument checks."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_device  # noqa: E402
import mini_xarray as mx  # noqa: E402
import pet_host_build as H  # noqa: E402
from oracle import pet_oracle as O  # noqa: E402
from xclim_b200 import Field, TimeAxis, _lib, converters, device, indices, set_options  # noqa: E402

LATS = np.array([-90.0, -78.5, -66.6, -45.0, -12.3, 0.0, 7.0, 45.0, 66.5, 66.6, 70.0, 89.9, 90.0])
K = 273.15


def _f32(x):
    return np.asarray(x, dtype=np.float32)


# ------------------------------------------------------------------------------------ solar terms
@pytest.mark.parametrize("calendar,start,n", [("360_day", "2001-01-01", 360), ("noleap", "2001-01-01", 365),
                                              ("standard", "2000-01-01", 366)])
def test_solar_tables_match_oracle(calendar, start, n):
    ta = TimeAxis.daily(start, n, calendar)
    for method, sc, scale in (("BR65", 1361.0, 1 / 41840.0), ("HG85", 1361.0, 1e-6 * 0.408), ("MB05", 1367.0, 1.0)):
        got = converters._daily_table(method, ta, LATS)
        ref = O.radiation_table(ta.year, ta.doy, calendar, LATS, sc) * scale
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-9 * np.abs(ref).max())
    # polar night gives 0, polar day a positive radiation; day lengths NaN there
    rad = converters._daily_table("MB05", ta, LATS)
    assert (rad[:, LATS == 90.0] >= 0).all() and (rad[:, LATS == 90.0] == 0).any() and (rad[:, LATS == 90.0] > 0).any()
    da = converters.day_angle(ta.year, ta.doy, calendar)[:, None]
    dl = converters.day_lengths(da, LATS[None, :])
    ref = np.array([[O.day_length(int(y), int(d), calendar, la) for la in LATS] for y, d in zip(ta.year, ta.doy)])
    np.testing.assert_array_equal(np.isnan(dl), np.isnan(ref))
    np.testing.assert_allclose(dl, ref, rtol=1e-12)
    assert np.isnan(dl[:, LATS == 90.0]).all() and not np.isnan(dl[:, LATS == 0.0]).any()


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pet.npz")


@pytest.mark.parametrize("calendar,start", [("360_day", "2001-01-01"), ("noleap", "2001-01-01"),
                                            ("standard", "2000-01-01")])
def test_solar_terms_match_reference_goldens(calendar, start):
    """The reference's own extraterrestrial_solar_radiation (its numba sunlit integral included) and day_lengths on
    every day of the year: the host tables bit for bit, the oracle within 1e-12."""
    g = np.load(GOLDEN)
    lats = g["lats"]
    r1361, r1367, dl = g[f"rad1361_{calendar}"], g[f"rad1367_{calendar}"], g[f"daylen_{calendar}"]
    ta = TimeAxis.daily(start, r1361.shape[0], calendar)
    assert int(g[f"year_{calendar}"]) == ta.year[0] and lats.min() == -90 and lats.max() == 90 and 0 in lats
    np.testing.assert_array_equal(converters._daily_table("MB05", ta, lats), r1367)
    np.testing.assert_array_equal(converters._daily_table("BR65", ta, lats), r1361 * (1 / 41840.0))
    np.testing.assert_array_equal(converters._daily_table("HG85", ta, lats), r1361 * 1e-6 * 0.408)
    da = converters.day_angle(ta.year, ta.doy, calendar)[:, None]
    np.testing.assert_array_equal(converters.day_lengths(da, lats[None, :]), dl)
    assert np.isnan(dl).any() and (r1361 == 0).any()          # polar nights and days are in the cases
    ref = O.radiation_table(ta.year, ta.doy, calendar, lats)
    np.testing.assert_allclose(ref, r1361, rtol=1e-12, atol=1e-9 * r1361.max())
    odl = np.array([[O.day_length(int(y), int(d), calendar, la) for la in lats] for y, d in zip(ta.year, ta.doy)])
    np.testing.assert_array_equal(np.isnan(odl), np.isnan(dl))
    np.testing.assert_allclose(odl, dl, rtol=1e-12)


# ------------------------------------------------------------------------------------ host build vs oracle
def _hostile(T, C, rng, lo, hi):
    x = rng.uniform(lo, hi, (T, C)).astype(np.float32)
    x[0, 0], x[1, 1 % C], x[2, 2 % C] = np.nan, np.inf, -np.inf
    return x


def _inputs(**kw):
    return [kw.get(n) for n in _lib.PET_INPUTS]


@pytest.mark.parametrize("method", ["BR65", "HG85", "MB05", "allen98"])
@pytest.mark.parametrize("wb", [False, True])
def test_host_build_daily_matches_oracle(method, wb):
    rng = np.random.default_rng(7)
    ta = TimeAxis.daily("2000-06-15", 40, "standard")       # June solstice: polar day and night
    T, C = len(ta), LATS.size
    tn = _hostile(T, C, rng, -20, 25)
    tx = (tn + rng.uniform(-3, 15, (T, C))).astype(np.float32)         # tasmax < tasmin on some days
    if method == "BR65":
        tn, tx = (tn * np.float32(1.8) + np.float32(32)), (tx * np.float32(1.8) + np.float32(32))
    kw = dict(tasmin=tn, tasmax=tx)
    if method == "allen98":
        kw.update(hurs=rng.uniform(0.1, 1, (T, C)).astype(np.float32), rsds=rng.uniform(0, 400, (T, C)).astype(np.float32),
                  rsus=rng.uniform(0, 80, (T, C)).astype(np.float32), rlds=rng.uniform(200, 400, (T, C)).astype(np.float32),
                  rlus=rng.uniform(200, 450, (T, C)).astype(np.float32), sfcWind=_hostile(T, C, rng, 0, 15))
    pr = rng.uniform(0, 5e-4, (T, C)).astype(np.float32) if wb else None
    lat_u, idx = np.unique(LATS, return_inverse=True)
    table = None if method == "allen98" else converters._daily_table(method, ta, lat_u)
    got = H.daily(_inputs(pr=pr, **kw), table, None if table is None else idx, H.params(method, wb))
    rad = None if table is None else table[:, idx]
    ref = _f32(O.daily_rate(O.daily_pet(method, rad, **kw), pr))
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    if method == "allen98":     # exp / log of the host libm against numpy's
        np.testing.assert_array_max_ulp(got[np.isfinite(ref)], ref[np.isfinite(ref)], maxulp=1)
    else:
        np.testing.assert_array_equal(got, ref)
    if method == "HG85":
        assert np.isnan(got[(tx < tn) & np.isfinite(tx) & np.isfinite(tn)]).all() or wb


@pytest.mark.parametrize("method", ["TW48", "DA02"])
@pytest.mark.parametrize("calendar,start,n", [("standard", "1999-11-17", 500), ("360_day", "2001-02-03", 400),
                                              ("noleap", "2003-12-31", 70)])
def test_host_build_monthly_matches_oracle(method, calendar, start, n):
    rng = np.random.default_rng(3)
    ta = TimeAxis.daily(start, n, calendar)
    lats = np.array([-70.0, 0.0, 45.0, 45.0, 80.0])
    T, C = len(ta), lats.size
    tas = rng.uniform(-10, 30, (T, C)).astype(np.float32)
    tas[:, 4] = -5                                        # heat index 0: NaN
    tas[40:80, 1] = np.nan                                # an all-NaN month
    tn = (tas - rng.uniform(0, 8, (T, C))).astype(np.float32)
    tx = (tas + rng.uniform(0, 8, (T, C))).astype(np.float32)
    pr = rng.uniform(0, 200, (T, C)).astype(np.float32)
    lat_u, idx = np.unique(lats, return_inverse=True)
    moff, yoff, ym, mdays = converters._months(ta)
    table = converters._monthly_table(method, ta, ym, lat_u)
    if method == "DA02":
        got = H.monthly(_inputs(tasmin=tn, tasmax=tx, pr=pr), moff, yoff, mdays, table, idx, H.params("DA02"))
        ref = O.monthly_pet("DA02", ta.year, ta.month, ta.doy, calendar, lats, tasmin=tn, tasmax=tx, pr=pr)
    else:
        wb = (pr * np.float32(1e-6)).astype(np.float32)
        got = H.monthly(_inputs(tas=tas, pr=wb), moff, yoff, mdays, table, idx, H.params("TW48", True))
        ref = O.monthly_pet("TW48", ta.year, ta.month, ta.doy, calendar, lats, tas=tas, wb_pr=wb)
    ref = _f32(ref)
    assert got.shape == ref.shape == (len(ym), C)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    np.testing.assert_array_max_ulp(got[np.isfinite(ref)], ref[np.isfinite(ref)], maxulp=1)
    if method == "TW48":
        assert np.isnan(got[:, 4]).all()


def test_host_build_monthly_group_longer_than_a_year_is_nan():
    """A C-ABI caller may pass YS groups of any size; more than 12 months gives NaN, not an overrun."""
    ta = TimeAxis.daily("2001-01-01", 400, "noleap")
    moff, _, ym, mdays = converters._months(ta)
    M = len(ym)
    tas = np.full((400, 2), 10.0, np.float32)
    table = converters._monthly_table("TW48", ta, ym, np.array([45.0]))
    out = H.monthly(_inputs(tas=tas), moff, np.array([0, M], np.int32), mdays, table, np.zeros(2, np.int32),
                    H.params("TW48"))
    assert M > 12 and np.isnan(out).all()


def test_parameter_struct_layout_agrees():
    """The product's ctypes struct (xclim_b200/_lib.py) lays XcPetParams out as the C compiler does (128 bytes;
    the doubles after the two ints and the 2 x 11 floats)."""
    P, c = _lib.PetParams, (ctypes.c_int64 * 3)()
    H.load().pet_host_params_layout(c)           # sizeof, offsetof in_scale, offsetof peta
    assert (ctypes.sizeof(P), P.in_scale.offset, P.peta.offset) == tuple(c) == (128, 8, 96)


# ------------------------------------------------------------------------------------ host layer
def _stand_in_daily(inputs, table, lat_index, params):
    np_in = [None if x is None else x.numpy() for x in inputs]
    out = H.daily(np_in, None if table is None else table.numpy(), None if lat_index is None else lat_index.numpy(),
                  params)
    return torch.from_numpy(out)


def _stand_in_monthly(inputs, moff, yoff, mdays, table, lat_index, params):
    np_in = [None if x is None else x.numpy() for x in inputs]
    return torch.from_numpy(H.monthly(np_in, moff, yoff, mdays, table.numpy(), lat_index.numpy(), params))


@pytest.fixture
def fake(monkeypatch):
    fake_device.install(monkeypatch)
    monkeypatch.setattr(device, "pet_daily", _stand_in_daily)
    monkeypatch.setattr(device, "pet_monthly", _stand_in_monthly)


def _field(values, units, start="2000-07-01", calendar="standard", lat=(45.0,), coord=True):
    v = np.asarray(values, dtype=np.float32)
    v = np.repeat(v[:, None], len(lat), axis=1)
    return Field(v, ("time", "lat"), TimeAxis.daily(start, v.shape[0], calendar), {"lat": np.asarray(lat)} if coord
                 else {}, {"units": units})


def _monthly_daily(values, units, start="1990-01-01", calendar="standard", **kw):
    """A daily series whose monthly means are ``values``, from the first of a month."""
    ta = TimeAxis.daily(start, 400, calendar)
    poff = ta.period_offsets("MS")[: len(values) + 1]
    daily = np.concatenate([np.full(poff[i + 1] - poff[i], v, np.float32) for i, v in enumerate(values)])
    return _field(daily, units, start=start, calendar=calendar, **kw)


TN, TX, TM = np.array([0, 5, 10]) + K, np.array([10, 15, 20]) + K, np.array([5, 10, 15]) + K


def test_known_answers_daily(fake):
    tn, tx, tm = _field(TN, "K"), _field(TX, "K"), _field(TM, "K")
    lat = np.array([45.0])
    out = indices.potential_evapotranspiration(tn, tx, lat=lat, method="BR65")
    np.testing.assert_allclose(out.values[2, 0], 3.861079 / 86400, rtol=1e-2)
    assert out.attrs["units"] == "kg m-2 s-1" and out.values.dtype == np.float32 and out.dims == ("time", "lat")
    out = indices.potential_evapotranspiration(tn, tx, tm, lat=lat, method="HG85")
    np.testing.assert_allclose(out.values[2, 0], 4.030339 / 86400, rtol=1e-2)
    out = indices.potential_evapotranspiration(tn, tx, lat=lat, method="MB05")
    np.testing.assert_allclose(out.values[2, 0], 2.78253138816 / 86400, rtol=1e-2)
    out = indices.potential_evapotranspiration(
        tn, tx, tm, lat=lat, hurs=_field([80, 70, 73], "%"), rsds=_field([43.09, 43.57, 70.20], "W m-2"),
        rsus=_field([12.51, 14.46, 20.36], "W m-2"), rlds=_field([293.65, 228.96, 275.40], "W m-2"),
        rlus=_field([311.39, 280.50, 311.30], "W m-2"), sfcWind=_field([14.11, 15.27, 10.70], "km h-1"),
        method="FAO_PM98")
    np.testing.assert_allclose(out.values[2, 0], 1.208832768 / 86400, rtol=1e-2)


def test_known_answers_monthly_from_daily(fake):
    out = indices.potential_evapotranspiration(tas=_monthly_daily(np.ones(12), "degC"), method="TW48")
    assert out.values.shape == (12, 1) and out.dims == ("time", "lat")
    np.testing.assert_allclose(out.values[1, 0], 42.7619242 / (86400 * 30), rtol=1e-1)
    out = indices.potential_evapotranspiration(
        tasmin=_monthly_daily([0, 5, 10], "degC"), tasmax=_monthly_daily([10, 15, 20], "degC"),
        tas=_monthly_daily([5, 10, 15], "degC"), pr=_monthly_daily([30, 0, 60], "mm/month"), lat=[45.0],
        method="DA02")
    np.testing.assert_allclose(out.values[2, 0], 2.32659206 / 86400, rtol=1e-2)


def test_known_answers_water_budget(fake):
    pr = _field([10, 10, 10], "mm/day")
    tn, tx = _field(TN, "K"), _field(TX, "K")
    out = indices.water_budget(pr, tasmin=tn, tasmax=tx, lat=[45.0], method="BR65")
    np.testing.assert_allclose(out.values[2, 0], 6.138921 / 86400, rtol=2e-3)
    out = indices.water_budget(pr, tasmin=tn, tasmax=tx, lat=[45.0], method="HG85")
    np.testing.assert_allclose(out.values[2, 0], 5.969661 / 86400, rtol=2e-3)
    out = indices.water_budget(_monthly_daily(np.ones(12) * 10, "mm/day"), tas=_monthly_daily(np.ones(12), "degC"),
                               method="TW48")
    np.testing.assert_allclose(out.values[1, 0], 8.5746025 / 86400, rtol=2e-1)
    assert out.attrs["units"] == "kg m-2 s-1"
    out = indices.water_budget(_field([10, 10, 10], "mm/day"), evspsblpot=_field([0, 10, 20], "mm/day"))
    np.testing.assert_allclose(out.values[:, 0], [10 / 86400, 0, -10 / 86400], rtol=1e-5, atol=1e-12)


def test_aliases_units_and_ms_labels(fake):
    tn, tx = _field(TN, "K"), _field(TX, "K")
    tnc, txc = _field(TN - K, "degC"), _field(TX - K, "degC")
    for a, b in (("BR65", "baierrobertson65"), ("HG85", "hargreaves85"), ("MB05", "mcguinnessbordne05"),
                 ("TW48", "thornthwaite48")):
        x = indices.potential_evapotranspiration(tn, tx, method=a).values
        np.testing.assert_array_equal(x, indices.potential_evapotranspiration(tn, tx, method=b).values)
        np.testing.assert_allclose(indices.potential_evapotranspiration(tnc, txc, method=a).values, x, rtol=1e-5)
    out = indices.potential_evapotranspiration(tn, tx, method="TW48")
    assert out.values.shape == (1, 1) and [str(t) for t in out.coords["time"]] == ["2000-07-01"]
    m = indices.potential_evapotranspiration(tas=_field(np.full(70, 280.0), "K", start="2001-01-20"), method="TW48")
    assert m.values.shape == (3, 1)
    assert [str(t) for t in m.coords["time"]] == ["2001-01-01", "2001-02-01", "2001-03-01"]


def test_lat_forms(fake):
    lats = (10.0, 45.0, -60.0)
    tn = _field(np.linspace(270, 280, 30), "K", lat=lats)
    tx = _field(np.linspace(280, 295, 30), "K", lat=lats)
    implicit = indices.potential_evapotranspiration(tn, tx, method="HG85").values
    np.testing.assert_array_equal(indices.potential_evapotranspiration(tn, tx, lat=np.array(lats), method="HG85").values,
                                  implicit)
    np.testing.assert_array_equal(
        indices.potential_evapotranspiration(tn, tx, lat=Field(np.array(lats), ("lat",)), method="HG85").values,
        implicit)
    scalar = indices.potential_evapotranspiration(tn, tx, lat=45.0, method="HG85").values
    np.testing.assert_array_equal(scalar[:, 1], implicit[:, 1])
    assert not np.array_equal(scalar[:, 0], implicit[:, 0])
    nolat = _field(np.linspace(270, 280, 30), "K", lat=lats, coord=False)
    with pytest.raises(ValueError, match="could not find latitude coordinate"):
        indices.potential_evapotranspiration(nolat, nolat, method="BR65")


def test_mini_xarray_in_and_out(fake, monkeypatch):
    mx.install(monkeypatch)
    T = 400
    t = np.arange(T)
    tas = (285 + 10 * np.sin(2 * np.pi * t / 365))[:, None, None] + np.zeros((1, 3, 2))
    tn, tx = mx.daily(tas - 4, "2001-01-15"), mx.daily(tas + 4, "2001-01-15")
    br = indices.potential_evapotranspiration(tn, tx, method="BR65")
    assert isinstance(br, mx.DataArray) and br.dims == ("time", "lat", "lon") and br.values.shape == (T, 3, 2)
    assert br.attrs["units"] == "kg m-2 s-1"
    ref = indices.potential_evapotranspiration(Field(np.asarray(tn.values, np.float32), ("time", "lat", "lon"),
                                                     TimeAxis.daily("2001-01-15", T, "noleap"),
                                                     {"lat": np.arange(3) * 0.25}, {"units": "K"}),
                                               Field(np.asarray(tx.values, np.float32), ("time", "lat", "lon"),
                                                     TimeAxis.daily("2001-01-15", T, "noleap"),
                                                     {"lat": np.arange(3) * 0.25}, {"units": "K"}), method="BR65")
    np.testing.assert_array_equal(np.asarray(br.values), ref.values)
    tw = indices.potential_evapotranspiration(tas=mx.daily(tas, "2001-01-15"), method="TW48")
    assert isinstance(tw, mx.DataArray) and tw.dims == ("time", "lat", "lon") and tw.values.shape == (14, 3, 2)
    labels = [str(v) for v in np.asarray(tw.coords["time"].values if hasattr(tw.coords["time"], "values")
                                         else tw.coords["time"])]
    assert labels[:3] == ["2001-01-01", "2001-02-01", "2001-03-01"] and labels[-1] == "2002-02-01"


def test_device_outputs_keep_tensors(fake):
    with set_options(device_outputs=True):
        out = indices.potential_evapotranspiration(_field(TN, "K"), _field(TX, "K"), method="BR65")
    assert isinstance(out.values, torch.Tensor)


def test_errors(fake):
    tn, tx = _field(TN, "K"), _field(TX, "K")
    with pytest.raises(NotImplementedError, match="'nope' method is not implemented."):
        indices.potential_evapotranspiration(tn, tx, method="nope")
    with pytest.raises(ValueError, match="Wind speed is required for Allen98 method."):
        indices.potential_evapotranspiration(tn, tx, method="allen98")
    with pytest.raises(ValueError, match="`tasmax`"):
        indices.potential_evapotranspiration(tn, method="BR65")
    with pytest.raises(ValueError, match="`pr`"):
        indices.potential_evapotranspiration(tn, tx, method="DA02")
    with pytest.raises(ValueError, match="DA02"):
        indices.water_budget(_field([1, 1, 1], "mm/d"), tasmin=tn, tasmax=tx, method="DA02")
    gap = TimeAxis.daily("2000-07-01", 3, "standard")
    gap.doy[2] += 1
    gap.day[2] += 1
    bad = Field(np.full((3, 1), 280, np.float32), ("time", "lat"), gap, {"lat": np.array([45.0])}, {"units": "K"})
    with pytest.raises(NotImplementedError, match="daily"):
        indices.potential_evapotranspiration(bad, bad, method="BR65")


# ------------------------------------------------------------------------------------ C argument checks
def test_c_argument_checks():
    lib = _lib.load()
    x = np.zeros((4, 3), np.float32)
    ptr = x.ctypes.data_as(ctypes.c_void_p)
    out = np.zeros_like(x)
    tab = np.zeros((4, 1))
    li = np.zeros(3, np.int32)

    def call(method, slots, table=tab, T=4, C=3, ldx=3, wb=0):
        P = H.params(method, wb)
        arr = (ctypes.c_void_p * _lib.PET_INPUTS.__len__())(*[ptr if i in slots else None
                                                            for i in range(len(_lib.PET_INPUTS))])
        return lib.xc_pet_daily_f32(arr, T, C, ldx, None if table is None else table.ctypes.data, 1, li.ctypes.data,
                                    ctypes.byref(P), out.ctypes.data, None)

    assert call("BR65", {0}) == _lib.XC_ERR_INVALID                 # tasmax missing
    assert call("BR65", {0, 1}, table=None) == _lib.XC_ERR_INVALID  # no solar table
    assert call("BR65", {0, 1}, ldx=2) == _lib.XC_ERR_INVALID       # ldx < C
    assert call("BR65", {0, 1}, wb=1) == _lib.XC_ERR_INVALID        # water budget without pr
    assert call("TW48", {2}) == _lib.XC_ERR_INVALID                 # a monthly method in the daily entry
    assert call("allen98", {0, 1, 3, 4, 5, 6, 7}) == _lib.XC_ERR_INVALID   # no wind
    assert "required input" in lib.xc_last_error().decode()
