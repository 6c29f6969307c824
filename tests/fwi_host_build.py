"""TEST INFRASTRUCTURE: build and bind the host build of the fire-weather device code (tests/csrc/fwi_host.cpp)."""
import ctypes

import numpy as np

import host_build
from xclim_b200 import _lib as L

_vp, _i64, _i32, _f64 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_double
SIGNATURES = {
    "fwi_host_last_error": (ctypes.c_char_p, []),
    "fwi_host_f32": (_i32, [_vp] * 12 + [_i64, _i64, _i64, _vp] + [_vp] * 9),
    "fwi_host_elementwise_f32": (_i32, [_i32, _vp, _vp, _i64, _f64, _f64, _f64, _vp]),
    "fwi_host_np_mean": (ctypes.c_float, [_vp, _i32, _i32]),
    "fwi_host_params_layout": (None, [ctypes.POINTER(_i64)]),
}


def load():
    return host_build.load("fwi", "fwi_host.cpp", signatures=SIGNATURES)


DEFAULTS = dict(temp_start_thresh=12.0, temp_end_thresh=5.0, snow_thresh=0.01, temp_condition_days=3,
                snow_condition_days=3, carry_over_fraction=0.75, wetting_efficiency_fraction=0.75, dc_start=15,
                dmc_start=6, ffmc_start=85, prec_thresh=1.0, dc_dry_factor=5, dmc_dry_factor=2, snow_cover_days=60,
                snow_min_cover_frac=0.75, snow_min_mean_depth=0.1)


def params(season_method=None, overwintering=False, dry_start=None, initial_start_up=True, **kw):
    p = dict(DEFAULTS)
    p.update(kw)
    P = L.FwiParams()
    P.season_mode, P.overwintering = L.FWI_SEASONS[season_method], int(overwintering)
    P.dry_start = L.FWI_DRY_STARTS[dry_start]
    P.initial_start_up = int(initial_start_up)
    for k in ("temp_condition_days", "snow_condition_days", "snow_cover_days"):
        setattr(P, k, int(p[k]))
    for k in ("temp_start_thresh", "temp_end_thresh", "snow_thresh", "prec_thresh", "snow_min_mean_depth", "dc_start",
              "dmc_start", "ffmc_start", "dc_dry_factor", "dmc_dry_factor", "snow_min_cover_frac", "carry_over_fraction",
              "wetting_efficiency_fraction"):
        setattr(P, k, float(p[k]))
    P.min_dc = float(p["dc_start"])
    for i, (sc, of) in enumerate(p.get("in_affine", [(1.0, 0.0)] * 5)):
        P.in_scale[i], P.in_offset[i] = sc, of
    return P


def run(tas, pr, hurs, ws, snd, mth, lat, season_mask, dc0, dmc0, ffmc0, winter_pr, *, outputs, **kw):
    """Same call shape as oracle.fire_oracle.fire_weather_calc, on the host build of the device code."""
    lib = load()
    T, C = tas.shape
    keep = []

    def ptr(a, dtype):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype=dtype)
        keep.append(a)
        return a.ctypes.data_as(ctypes.c_void_p)

    out = {}
    optr = {}
    for name in ("DC", "DMC", "FFMC", "ISI", "BUI", "FWI", "DSR"):
        if name in outputs:
            out[name] = np.full((T, C), -777.0, np.float32)
            optr[name] = out[name].ctypes.data_as(ctypes.c_void_p)
        else:
            optr[name] = None
    mptr = wptr = None
    if "season_mask" in outputs:
        out["season_mask"] = np.full((T, C), 9, np.uint8)
        mptr = out["season_mask"].ctypes.data_as(ctypes.c_void_p)
    if "winter_pr" in outputs:
        out["winter_pr"] = np.full(C, -777.0, np.float32)
        wptr = out["winter_pr"].ctypes.data_as(ctypes.c_void_p)
    P = params(**kw)
    st = lib.fwi_host_f32(ptr(tas, np.float32), ptr(pr, np.float32), ptr(hurs, np.float32), ptr(ws, np.float32),
                          ptr(snd, np.float32), ptr(season_mask, np.uint8), ptr(mth, np.int8), ptr(lat, np.float64),
                          ptr(dc0, np.float32), ptr(dmc0, np.float32), ptr(ffmc0, np.float32), ptr(winter_pr, np.float32),
                          ctypes.c_int64(T), ctypes.c_int64(C), ctypes.c_int64(C), ctypes.byref(P),
                          optr["DC"], optr["DMC"], optr["FFMC"], optr["ISI"], optr["BUI"], optr["FWI"], optr["DSR"],
                          mptr, wptr)
    if st != 0:
        raise ValueError(lib.fwi_host_last_error().decode())
    if "season_mask" in out:
        out["season_mask"] = out["season_mask"].astype(bool)
    return out


def elementwise(kind, a, b=None, p=(0.0, 0.0, 0.0)):
    """The element-wise entry point on the host build (kind: ISI, BUI, FWI, DSR, OWDC)."""
    lib = load()
    a = np.ascontiguousarray(a, dtype=np.float32)
    bb = None if b is None else np.ascontiguousarray(np.broadcast_to(b, a.shape), dtype=np.float32)
    out = np.empty_like(a)
    lib.fwi_host_elementwise_f32(ctypes.c_int32(L.FWI_ELEMENTWISE[kind]), a.ctypes.data_as(ctypes.c_void_p),
                                 None if bb is None else bb.ctypes.data_as(ctypes.c_void_p), ctypes.c_int64(a.size),
                                 ctypes.c_double(p[0]), ctypes.c_double(p[1]), ctypes.c_double(p[2]),
                                 out.ctypes.data_as(ctypes.c_void_p))
    return out
