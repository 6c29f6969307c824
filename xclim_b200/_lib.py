"""ctypes binding of ``libxclim_b200.so`` (the C ABI declared in ``include/xclim_b200.h``).

There is NO CPU fallback: if the shared library is missing or a call fails, this raises.
"""
from __future__ import annotations

import ctypes as C
import os

from ._build import LIB_PATH

# status codes (include/xclim_b200.h)
XC_OK, XC_ERR_INVALID, XC_ERR_UNSUPPORTED, XC_ERR_CUDA = 0, -1, -2, -3

OPS = {">": 0, "gt": 0, "<": 1, "lt": 1, ">=": 2, "ge": 2, "<=": 3, "le": 3, "==": 4, "eq": 4, "!=": 5, "ne": 5}
OP_ISNAN, OP_NOTNAN = 6, 7
RL_REDUCERS = {"max": 0, "min": 1, "sum": 2, "count": 3, "mean": 4, "std": 5}
STATS = {"sum": 0, "integral": 0, "mean": 1, "min": 2, "max": 3, "std": 4, "var": 5, "count": 6}
TF_NONE, TF_EXCESS, TF_WHERE = 0, 1, 2

_i32, _i64, _f64, _u64, _vp = C.c_int32, C.c_int64, C.c_double, C.c_uint64, C.c_void_p

#: symbol -> (restype, argtypes); must list every function declared in include/xclim_b200.h
SIGNATURES = {
    "xc_version": (_i32, []),
    "xc_last_error": (C.c_char_p, []),
    "xc_device_sm_count": (_i32, [C.POINTER(_i32)]),
    "xc_period_count_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _i32, _f64, _i32, _vp, _vp, _vp]),
    "xc_period_runstat_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _i32, _f64, _i32, _i32, _i32, _i32,
                                     _vp, _vp, _vp]),
    "xc_period_runstat2_f32": (_i32, [_vp, _vp, _i64, _i64, _i64, _vp, _i32, _i32, _f64, _i32, _f64, _i32, _i32, _i32,
                                      _i32, _vp, _vp]),
    "xc_period_run_quantile_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _i32, _i32, _f64, _i32, _f64, _i32, _i32,
                                          _vp, _vp]),
    "xc_period_run_maxsum_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _i32, _f64, _i32, _i32, _vp, _vp]),
    "xc_period_boundary_run_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _i32, _f64, _i32, _i32, _i32, _vp, _vp]),
    "xc_period_boundary_run_range_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _vp, _i32, _i32, _f64, _i32, _i32,
                                                _i32, _i32, _vp, _vp, _vp]),
    "xc_period_runstat_gap_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _i32, _f64, _i32, _i32, _i32, _i32, _vp, _vp]),
    "xc_period_reduce_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _i32, _i32, _i32, _f64, _vp, _vp, _vp]),
    "xc_rolling_period_reduce_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "xc_rolling_period_reduce_sel_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "xc_spell_runstat_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _i32, _i32, _i32, _f64, _i32, _i32, _vp, _vp]),
    "xc_spell_mask_f32": (_i32, [_vp, _i64, _i64, _i64, _i32, _i32, _i32, _f64, _vp, _i32, _vp, _vp]),
    "xc_spell_sum_interval": (_i32, [_i32, _f64, _i32, _i32, _vp, _vp, _vp]),
    "xc_percentile_doy_workspace_bytes": (_i64, [_i64, _i64, _i32, _i32, _i32, _i32]),
    "xc_percentile_doy_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _i32, _i32, _i32, _vp, _i32, _f64, _f64,
                                     _vp, _vp, _i64, _vp]),
    "xc_percentile_doy_vrow_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _i32, _f64,
                                          _f64, _vp, _vp, _i64, _vp]),
    "xc_percentile_doy_generic_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _i32, _i32, _i32, _f64, _f64, _f64,
                                             _vp, _vp, _i64, _vp]),
    "xc_doy_interp_f64": (_i32, [_vp, _i32, _i64, _i32, _i32, _vp, _vp]),
    "xc_doy_threshold_count_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _i32, _i32, _vp, _vp, _vp]),
    "xc_doy_threshold_count_years_f32": (_i32, [_vp, _i64, _i64, _i64, _i64, _i32, _i32, _vp, _i32, _vp, _vp, _vp]),
    "xc_doy_runstat_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp,
                                  _vp]),
    "xc_period_sums_thr_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _i64, _i32, _f64, _vp, _vp, _vp]),
    "xc_doy_count2_f32": (_i32, [_vp, _vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "xc_period_range_stat_f32": (_i32, [_vp, _vp, _i64, _i64, _i64, _vp, _i32, _i32, _i32, _vp, _vp]),
    "xc_bootstrap_doy_count_f32": (_i32, [_vp, _i64, _i64, _i64, _i64, _i32, _i32, _vp, _i32, _i32, _f64, _f64,
                                          _f64, _i32, _vp, _vp, _vp]),
    "xc_bootstrap_doy_index_scratch_bytes": (_i64, [_i32, _i32, _i64]),
    "xc_bootstrap_doy_index_f32": (_i32, [_vp, _i64, _i64, _i64, _i64, _i32, _i32, _vp, _i32, _i32, _f64, _f64, _f64,
                                          _i32, _i32, _i32, _i32, _f64, _vp, _vp, _i64, _vp, _vp]),
    "xc_eqm_train_workspace_bytes": (_i64, [_i64, _i64, _i32]),
    "xc_eqm_train_f32": (_i32, [_vp, _vp, _i64, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _i64, _vp]),
    "xc_eqm_adjust_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "xc_qdm_adjust_workspace_bytes": (_i64, [_i64, _i64]),
    "xc_qdm_adjust_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _i64, _vp]),
    "xc_dqm_train_workspace_bytes": (_i64, [_i64, _i64, _i32]),
    "xc_dqm_train_f32": (_i32, [_vp, _vp, _i64, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _i64, _vp]),
    "xc_poly_fit_f32": (_i32, [_vp, _i64, _i64, _i64, _i32, _i32, _vp, _vp, _vp]),
    "xc_dqm_adjust_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "xc_detrend_apply_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp]),
    "xc_synth_f32": (_i32, [_vp, _i64, _i64, _i64, _i64, _i64, _i64, _i32, _i32, _u64, _vp]),
    "xc_mask_steps_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _vp]),
    "xc_host_stream_workspace_bytes": (_i64, [_i64, _i64, _vp, _i32]),
    "xc_period_count_arr_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _i32, _vp, _i64, _vp, _vp]),
    "xc_period_multi_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _i32, _vp]),
    "xc_table_cell_major_f64": (_i32, [_vp, _i32, _i32, _i64, _vp, _vp]),
    "xc_host_pinned": (_i32, [_vp]),
    "xc_copy_box_async": (_i32, [_vp, _i64, _vp, _i64, _i64, _i64, _i32, _vp]),
    "xc_fwi_f32": (_i32, [_vp] * 12 + [_i64, _i64, _i64, _vp] + [_vp] * 9 + [_vp]),
    "xc_fwi_elementwise_f32": (_i32, [_i32, _vp, _vp, _i64, _f64, _f64, _f64, _vp, _vp]),
    "xc_period_runstat_f32_host": (_i32, [_vp, _i64, _i64, _vp, _i32, _i32, _f64, _i32, _i32, _i32, _vp, _vp,
                                          _vp, _i64]),
    "xc_rolling_mean_f32": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _i64, _vp]),
    "xc_si_fit_workspace_bytes": (_i64, [_i64, _i32]),
    "xc_si_fit_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _f64, _vp, _vp, _vp, _vp,
                             _vp, _i64, _vp]),
    "xc_si_apply_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _vp, _i32, _i32, _f64, _f64, _f64, _vp,
                               _i64, _vp]),
    "xc_ev_fit_workspace_bytes": (_i64, [_i64, _i64]),
    "xc_ev_fit_f32": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _vp, _vp, _i64, _vp]),
    "xc_ev_transform_f64": (_i32, [_vp, _i64, _i32, _i32, _vp, _i32, _vp, _vp]),
    "xc_analog_f32": (_i32, [_vp, _i64, _i64, _vp, _i64, _i64, _i64, _i64, _i32, _f64, _vp, _vp, _vp, _vp]),
    "xc_pet_daily_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i64, _vp, _vp, _vp, _vp]),
    "xc_pet_monthly_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "xc_ens_percentiles_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _f64, _f64, _i32, _vp, _vp]),
    "xc_ens_moments_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    "xc_ens_robustness_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i64, _i64, _i64, _vp, _i64, _i64, _vp, _i64, _i64,
                                     _vp, _i32, _f64, _i32, _vp, _vp, _vp]),
    "xc_chill_daily_f32": (_i32, [_vp, _vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _i32, _vp, _f64, _f64, _f64, _f64,
                                  _i32, _vp, _vp, _vp, _vp]),
    "xc_chill_hourly": (_i32, [_vp, _i32, _i64, _i64, _i64, _vp, _i32, _vp, _f64, _f64, _f64, _f64, _i32, _vp, _vp,
                               _vp, _vp]),
    "xc_hourly_temperature_f32": (_i32, [_vp, _vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _vp]),
    "xc_rain_season_f32": (_i32, [_vp, _i64, _i64, _i64, _vp, _i32, _vp, C.c_float, _f64, _i32, _i32, _f64, _i32,
                                  _i32, _f64, _i32, _i32, _vp, _vp, _vp]),
}

# ensembles (include/xclim_b200.h e1)
ENS_MAX_MEMBERS, ENS_MAX_PER = 128, 32
ENS_TESTS = {None: 0, "abs_thresh": 1, "rel_thresh": 2, "ttest": 3, "welch-ttest": 4, "ipcc-ar6-c": 5}
ENS_FRACTIONS = ("changed", "positive", "changed_positive", "negative", "changed_negative", "valid", "agree")

# standardized indices (include/xclim_b200.h s1)
SI_DISTS = {"gamma": 0, "fisk": 1, "lognorm": 2}
SI_METHODS = {"APP": 0, "ML": 1}
SI_STATUS_FITDATA, SI_STATUS_ROOT_NAN, SI_STATUS_ROOT_SIGN, SI_STATUS_LOGNORM_FALLBACK = 1, 2, 4, 8

# frequency analysis (include/xclim_b200.h s2)
EV_DISTS = {"norm": 0, "gumbel_r": 1, "genextreme": 2}
EV_KINDS = {"ppf": 0, "isf": 1, "cdf": 2}
EV_STATUS_NOT_CONVERGED, EV_STATUS_UNBOUNDED, EV_STATUS_ROOT_NAN, EV_STATUS_ROOT_SIGN = 1, 2, 4, 8

# spatial analogues (include/xclim_b200.h a1)
AN_METHODS = {"seuclidean": 0, "nearest_neighbor": 1, "zech_aslan": 2, "szekely_rizzo": 3, "kolmogorov_smirnov": 4,
              "kldiv": 5, "mahalanobis": 6}
AN_MAX_D, AN_KLDIV_MAX_K = 16, 16
AN_STATUS_NOT_FINITE, AN_STATUS_CHKFINITE = 1, 2

# potential evapotranspiration (include/xclim_b200.h p1)
PET_METHODS = {"BR65": 0, "HG85": 1, "MB05": 2, "allen98": 3, "TW48": 4, "DA02": 5, "given": 6}
PET_MONTHLY = ("TW48", "DA02")
PET_INPUTS = ("tasmin", "tasmax", "tas", "hurs", "rsds", "rsus", "rlds", "rlus", "sfcWind", "pr", "evspsblpot")


# chill portions and units (include/xclim_b200.h c1)
CHILL_ROW = 28
CHILL_PORTIONS, CHILL_UNITS, CHILL_POSITIVE_ONLY = 1, 2, 4

# rain season (include/xclim_b200.h r1)
RS_METHODS = {"per_day": 0, "total": 1}
RS_PRE, RS_START, RS_END = 1, 2, 4
RS_MAX_WINDOW = 64


class PetParams(C.Structure):
    """include/xclim_b200.h XcPetParams."""
    _fields_ = [("method", _i32), ("water_budget", _i32), ("in_scale", C.c_float * 11), ("in_offset", C.c_float * 11),
                ("peta", _f64), ("petb", _f64), ("wind_num", _f64), ("wind_den", _f64)]


# ---- plan of the fused multi-output pass (include/xclim_b200.h: XcMultiPlan)
MULTI_MAX_COND, MULTI_MAX_RUNS, MULTI_MAX_MSUM, MULTI_MAX_SUMS = 6, 4, 1, 3


class MultiCond(C.Structure):
    _fields_ = [("sgn", C.c_float), ("thr", C.c_float), ("wmax", _i32), ("slot_n", _i32), ("slot_max", _i32)]


class MultiRun(C.Structure):
    _fields_ = [("cond", _i32), ("window", _i32), ("kind", _i32), ("slot", _i32)]


class MultiMaxSum(C.Structure):
    _fields_ = [("cond", _i32), ("window", _i32), ("sgn", C.c_float), ("thr0", C.c_float), ("slot", _i32)]


class MultiSum(C.Structure):
    _fields_ = [("sgn", C.c_float), ("thr", C.c_float), ("off_sgn", C.c_float), ("off", C.c_float), ("mode", _i32),
                ("slot", _i32)]


class MultiPlan(C.Structure):
    _fields_ = [("n_cond", _i32), ("n_runs", _i32), ("n_msum", _i32), ("n_sums", _i32),
                ("cond", MultiCond * MULTI_MAX_COND), ("runs", MultiRun * MULTI_MAX_RUNS),
                ("msum", MultiMaxSum * MULTI_MAX_MSUM), ("sums", MultiSum * MULTI_MAX_SUMS),
                ("slot_sum", _i32), ("slot_mean", _i32), ("slot_min", _i32), ("slot_max", _i32)]


class FwiParams(C.Structure):
    """include/xclim_b200.h XcFwiParams."""
    _fields_ = ([(n, _i32) for n in ("season_mode", "overwintering", "dry_start", "initial_start_up",
                                     "temp_condition_days", "snow_condition_days", "snow_cover_days")]
                + [(n, C.c_float) for n in ("temp_start_thresh", "temp_end_thresh", "snow_thresh", "prec_thresh",
                                            "snow_min_mean_depth", "dc_start", "dmc_start", "ffmc_start",
                                            "dc_dry_factor", "dmc_dry_factor")]
                + [(n, _f64) for n in ("snow_min_cover_frac", "carry_over_fraction", "wetting_efficiency_fraction",
                                       "min_dc")]
                + [("in_scale", C.c_float * 5), ("in_offset", C.c_float * 5)])


FWI_ELEMENTWISE = {"ISI": 0, "BUI": 1, "FWI": 2, "DSR": 3, "OWDC": 4}
FWI_SEASONS = {None: 0, "mask": 1, "WF93": 2, "LA08": 3, "GFWED": 4}
FWI_DRY_STARTS = {None: 0, "CFS": 1, "GFWED": 2, "GFWED+SNOW": 3}

_lib = None


class XclimB200Error(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load the shared library (once).  Raises if it has not been built: no silent fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise XclimB200Error(
            f"{LIB_PATH} is missing: build it with `python -m xclim_b200._build` "
            "(the xclim_b200 hot path has no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int) -> None:
    """Translate a C-ABI status into the exception the reference raises for the same condition."""
    if status == XC_OK:
        return
    msg = load().xc_last_error().decode("utf-8", "replace")
    if status == XC_ERR_INVALID:
        raise ValueError(msg)
    if status == XC_ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    raise XclimB200Error(msg)


def op_code(op: str, constrain=None) -> int:
    """Operator name -> code with the validation of indices/generic.py:255-298 (`get_op`)."""
    if op in ("gteq", "lteq"):     # deprecated spellings, renamed with a warning (indices/generic.py:273-278)
        import warnings
        renamed = {"gteq": "ge", "lteq": "le"}[op]
        warnings.warn(f"`{op}` is being renamed `{renamed}` for compatibility.")
        op = renamed
    if op not in OPS:
        raise ValueError(f"Operation `{op}` not recognized.")
    if constrain:
        allowed = set()
        for c in ([constrain] if isinstance(constrain, str) else constrain):
            allowed.add(OPS[c])
        if OPS[op] not in allowed:
            raise ValueError(f"Operation `{op}` not permitted for indice.")
    return OPS[op]
