"""TEST INFRASTRUCTURE: build and bind the host build of the evapotranspiration device code
(tests/csrc/pet_host.cpp over xclim_b200/csrc/pet_core.cuh), behind the argument lists of device.pet_daily and
device.pet_monthly with numpy arrays in place of device tensors."""
import ctypes

import numpy as np

import host_build
from xclim_b200 import _lib as L

_vp, _i64, _i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32
SIGNATURES = {
    "pet_host_daily": (_i32, [_vp, _i64, _i64, _i64, _vp, _i64, _vp, _vp, _vp]),
    "pet_host_monthly": (_i32, [_vp, _i64, _i64, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _vp]),
    "pet_host_params_layout": (None, [ctypes.POINTER(_i64)]),
}


def load():
    return host_build.load("pet", "pet_host.cpp", signatures=SIGNATURES)


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _inputs(inputs):
    arrs = [None if x is None else np.ascontiguousarray(x, dtype=np.float32) for x in inputs]
    ref = next(x for x in arrs if x is not None)
    return arrs, (ctypes.c_void_p * len(arrs))(*[_p(x) for x in arrs]), ref.shape


def params(method, water_budget=False, affine=None, peta=0.00516409319477, petb=0.0874972822289):
    P = L.PetParams()
    P.method, P.water_budget = L.PET_METHODS[method], int(water_budget)
    for i in range(len(L.PET_INPUTS)):
        P.in_scale[i], P.in_offset[i] = (affine or {}).get(L.PET_INPUTS[i], (1.0, 0.0))
    P.peta, P.petb = peta, petb
    P.wind_num, P.wind_den = float(np.log(67.8 * 2 - 5.42)), float(np.log(67.8 * 10 - 5.42))
    return P


def daily(inputs, table, lat_index, P):
    """(T, C) float32 of the host build; ``inputs``: the XC_PET_N_IN (T, C) arrays or None.  Raises ValueError
    where the C ABI rejects the arguments."""
    keep, ptrs, (T, C) = _inputs(inputs)
    tab = None if table is None else np.ascontiguousarray(table, dtype=np.float64)
    li = None if lat_index is None else np.ascontiguousarray(lat_index, dtype=np.int32)
    out = np.full((T, C), np.nan, dtype=np.float32)
    st = load().pet_host_daily(ptrs, T, C, C, _p(tab), 0 if tab is None else tab.shape[1], _p(li),
                               ctypes.byref(P), _p(out))
    if st:
        raise ValueError("invalid arguments")
    return out


def monthly(inputs, moff, yoff, mdays, table, lat_index, P):
    keep, ptrs, (T, C) = _inputs(inputs)
    moff, yoff = np.ascontiguousarray(moff, np.int32), np.ascontiguousarray(yoff, np.int32)
    mdays, tab = np.ascontiguousarray(mdays, np.float64), np.ascontiguousarray(table, np.float64)
    li = np.ascontiguousarray(lat_index, np.int32)
    out = np.full((moff.size - 1, C), np.nan, dtype=np.float32)
    st = load().pet_host_monthly(ptrs, T, C, C, _p(moff), moff.size - 1, _p(yoff), yoff.size - 1, _p(mdays), _p(tab),
                                 tab.shape[1], _p(li), ctypes.byref(P), _p(out))
    if st:
        raise ValueError("invalid arguments")
    return out
