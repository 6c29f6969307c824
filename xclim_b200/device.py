"""Thin device layer: torch tensors for HBM buffers + ctypes calls into ``libxclim_b200.so``.

PyTorch is plumbing here (device memory, streams, pinned host staging); every computation is one
of the hand-written kernels behind the C ABI.  All functions take/return CUDA tensors laid out as
``(time, cell)`` float32 row-major -- the flattened view of the reference's ``(time, lat, lon)``.
"""
from __future__ import annotations

import warnings

import numpy as np
import torch

from . import _lib
from ._lib import check, load


def _require_cuda():
    if not torch.cuda.is_available():
        raise _lib.XclimB200Error("xclim_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")


def current_stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t) -> int | None:
    return None if t is None else t.data_ptr()


# ---------------------------------------------------------------------------------------- staging
def to_time_cell(values, time_axis: int, device=None):
    """Unwrap an array to a contiguous ``(T, C)`` float32 CUDA tensor.

    Returns ``(x2d, cell_shape)``.  numpy inputs are staged through pinned host memory; CUDA
    tensors already in ``(time, ...)`` float32 contiguous layout are used in place (zero copy).
    """
    _require_cuda()
    if isinstance(values, torch.Tensor):
        t = values
        if time_axis != 0:
            t = t.movedim(time_axis, 0)
        if t.dtype != torch.float32:
            t = t.to(torch.float32)
        if not t.is_cuda:
            t = t.contiguous().pin_memory().to(device or "cuda", non_blocking=True)
        t = t.contiguous()
    else:
        a = np.asarray(values)
        if time_axis != 0:
            a = np.moveaxis(a, time_axis, 0)
        if a.dtype != np.float32:
            if a.dtype.kind == "f":
                warnings.warn(f"xclim_b200 computes in float32: casting input from {a.dtype}", stacklevel=3)
            a = a.astype(np.float32)
        a = np.ascontiguousarray(a)
        h = torch.from_numpy(a)
        try:
            h = h.pin_memory()
        except RuntimeError:  # pragma: no cover - pinning can fail for huge buffers
            pass
        t = h.to(device or "cuda", non_blocking=True)
    cell_shape = tuple(t.shape[1:])
    return t.reshape(t.shape[0], -1), cell_shape


_small_cache: dict = {}


def dev_ints(arr, dtype, device) -> torch.Tensor:
    """Small integer index arrays (period offsets, doy index) cached per device."""
    a = np.ascontiguousarray(np.asarray(arr, dtype=dtype))
    key = (str(device), a.dtype.str, a.tobytes())
    t = _small_cache.get(key)
    if t is None:
        if len(_small_cache) > 256:
            _small_cache.clear()
        t = torch.from_numpy(a).to(device)
        _small_cache[key] = t
    return t


# ---------------------------------------------------------------------------------------- kernels
def period_count(x2d, poff, op_code, thr, cmp_f64=False, want_valid=False):
    T, C = x2d.shape
    P = len(poff) - 1
    poff_d = dev_ints(poff, np.int32, x2d.device)
    out = torch.empty((P, C), dtype=torch.int32, device=x2d.device)
    valid = torch.empty((P, C), dtype=torch.int32, device=x2d.device) if want_valid else None
    check(load().xc_period_count_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(), P, op_code,
                                     float(thr), int(bool(cmp_f64)), out.data_ptr(), _ptr(valid),
                                     current_stream_ptr()))
    return out, valid


def period_count_arr(x2d, poff, op_code, thr2d, per_time):
    """Counts against an array threshold: ``thr2d`` float64 ``(T, C)`` (per_time) or ``(1, C)`` (per cell)."""
    T, C = x2d.shape
    P = len(poff) - 1
    assert thr2d.dtype == torch.float64 and thr2d.is_contiguous() and thr2d.shape[-1] == C
    poff_d = dev_ints(poff, np.int32, x2d.device)
    out = torch.empty((P, C), dtype=torch.int32, device=x2d.device)
    check(load().xc_period_count_arr_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(), P, op_code,
                                         thr2d.data_ptr(), C if per_time else 0, out.data_ptr(), current_stream_ptr()))
    return out


def period_runstat(x2d, poff, op_code, thr, reducer_code, window, resample_before_rl=True, cmp_f64=False,
                   want_valid=False):
    T, C = x2d.shape
    P = len(poff) - 1
    poff_d = dev_ints(poff, np.int32, x2d.device)
    out = torch.empty((P, C), dtype=torch.float32, device=x2d.device)
    valid = torch.empty((P, C), dtype=torch.int32, device=x2d.device) if want_valid else None
    check(load().xc_period_runstat_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(), P, op_code,
                                       float(thr), int(bool(cmp_f64)), reducer_code, int(window),
                                       int(bool(resample_before_rl)), out.data_ptr(), _ptr(valid),
                                       current_stream_ptr()))
    return out, valid


def period_reduce(x2d, poff, stat_code, transform=0, op_code=0, thr=0.0, want_valid=False):
    T, C = x2d.shape
    P = len(poff) - 1
    poff_d = dev_ints(poff, np.int32, x2d.device)
    out = torch.empty((P, C), dtype=torch.float32, device=x2d.device)
    valid = torch.empty((P, C), dtype=torch.int32, device=x2d.device) if want_valid else None
    check(load().xc_period_reduce_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(), P, stat_code,
                                      transform, op_code, float(thr), out.data_ptr(), _ptr(valid),
                                      current_stream_ptr()))
    return out, valid


def synth(T, C, kind, seed, cell_offset=0, cells_per_lat=1440, n_lat_global=721, year_len=365, device="cuda"):
    """Synthetic (T, C) float32 input generated in HBM (kind 0 = pr mm/d, 1 = tasmax K)."""
    _require_cuda()
    out = torch.empty((T, C), dtype=torch.float32, device=device)
    check(load().xc_synth_f32(out.data_ptr(), T, C, C, cell_offset, cells_per_lat, n_lat_global, year_len,
                              kind, seed, current_stream_ptr()))
    return out


# ------------------------------------------------------------------------------------ percentiles
def percentile_doy(x2d, doy_index, year_index, n_doy, n_years, window, percentiles, alpha, beta,
                   force_generic=False, vrow=None):
    """(n_per, n_doy, C) float64 table of day-of-year percentiles (core/calendar.py:448-479).
    ``vrow`` (int32[T], -1 = missing): read the value of step t from row vrow[t] (bootstrap
    replacements on calendars with leap years)."""
    T, C = x2d.shape
    per = np.ascontiguousarray(np.atleast_1d(np.asarray(percentiles, dtype=np.float64)))
    doy = np.ascontiguousarray(np.asarray(doy_index, dtype=np.int16))
    yr = np.ascontiguousarray(np.asarray(year_index, dtype=np.int16))
    assert doy.size == T and yr.size == T
    lib = load()
    ws_bytes = int(lib.xc_percentile_doy_workspace_bytes(T, C, n_doy, n_years, window, per.size))
    ws = torch.empty(max(ws_bytes, 256), dtype=torch.uint8, device=x2d.device)
    out = torch.empty((per.size, n_doy, C), dtype=torch.float64, device=x2d.device)
    if force_generic:
        for i, p in enumerate(per):
            check(lib.xc_percentile_doy_generic_f32(x2d.data_ptr(), T, C, x2d.stride(0), doy.ctypes.data,
                                                    yr.ctypes.data, n_doy, n_years, int(window), float(p),
                                                    float(alpha), float(beta), out[i].data_ptr(), ws.data_ptr(),
                                                    ws.numel(), current_stream_ptr()))
    elif vrow is not None:
        vr = np.ascontiguousarray(np.asarray(vrow, dtype=np.int32))
        assert vr.size == T
        check(lib.xc_percentile_doy_vrow_f32(x2d.data_ptr(), T, C, x2d.stride(0), doy.ctypes.data, yr.ctypes.data,
                                             vr.ctypes.data, n_doy, n_years, int(window), per.ctypes.data, per.size,
                                             float(alpha), float(beta), out.data_ptr(), ws.data_ptr(), ws.numel(),
                                             current_stream_ptr()))
    else:
        check(lib.xc_percentile_doy_f32(x2d.data_ptr(), T, C, x2d.stride(0), doy.ctypes.data, yr.ctypes.data,
                                        n_doy, n_years, int(window), per.ctypes.data, per.size, float(alpha),
                                        float(beta), out.data_ptr(), ws.data_ptr(), ws.numel(),
                                        current_stream_ptr()))
    return out


def table_cell_major(table):
    """(n_per, n_doy, C) float64 doy-major table -> (C, n_doy, n_per), the reference's
    ``(*space, dayofyear, percentiles)`` order (core/calendar.py:479-483), transposed in HBM."""
    n_per, n_doy, C = table.shape
    assert table.dtype == torch.float64 and table.is_contiguous()
    out = torch.empty((C, n_doy, n_per), dtype=torch.float64, device=table.device)
    check(load().xc_table_cell_major_f64(table.data_ptr(), n_per, n_doy, C, out.data_ptr(), current_stream_ptr()))
    return out


def transpose_f64(m):
    """(A, B) float64 -> (B, A), tiled in shared memory (the layout kernel of table_cell_major with n_per = 1)."""
    A, B = m.shape
    assert m.dtype == torch.float64 and m.is_contiguous()
    out = torch.empty((B, A), dtype=torch.float64, device=m.device)
    check(load().xc_table_cell_major_f64(m.data_ptr(), 1, A, B, out.data_ptr(), current_stream_ptr()))
    return out


def doy_interp(table2d, doy_min, doy_max):
    """core/calendar.py:690-726 on a (n_src, C) float64 device table."""
    n_src, C = table2d.shape
    out = torch.empty((doy_max - doy_min + 1, C), dtype=torch.float64, device=table2d.device)
    check(load().xc_doy_interp_f64(table2d.data_ptr(), n_src, C, doy_min, doy_max, out.data_ptr(),
                                   current_stream_ptr()))
    return out


def doy_threshold_count(x2d, poff, doy_index, table2d, op_code, want_valid=False):
    """#{t in period : float64(x[t]) op table[doy[t]-1]} (indices/_multivariate.py:1583-1590)."""
    T, C = x2d.shape
    P = len(poff) - 1
    assert table2d.dtype == torch.float64 and table2d.is_contiguous() and table2d.shape[1] == C
    doy_index = np.asarray(doy_index)
    assert int(doy_index.max()) <= table2d.shape[0] and int(doy_index.min()) >= 1
    out = torch.empty((P, C), dtype=torch.int32, device=x2d.device)
    valid = torch.empty((P, C), dtype=torch.int32, device=x2d.device) if want_valid else None
    # whole years of equal length with doy == position in the year: the year-blocked kernel
    poff = np.asarray(poff)
    L = int(poff[1] - poff[0])
    if (op_code <= 3 and C % 4 == 0 and x2d.stride(0) % 4 == 0 and x2d.data_ptr() % 16 == 0
            and np.all(np.diff(poff) == L) and L == table2d.shape[0]
            and np.array_equal(doy_index[poff[0]:poff[-1]], np.tile(np.arange(1, L + 1), P))):
        check(load().xc_doy_threshold_count_years_f32(x2d.data_ptr(), T, C, x2d.stride(0), int(poff[0]), P, L,
                                                       table2d.data_ptr(), op_code, out.data_ptr(), _ptr(valid),
                                                       current_stream_ptr()))
        return out, valid
    poff_d = dev_ints(poff, np.int32, x2d.device)
    doy_d = dev_ints(doy_index, np.int16, x2d.device)
    check(load().xc_doy_threshold_count_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(), P,
                                            doy_d.data_ptr(), table2d.data_ptr(), table2d.shape[0], op_code,
                                            out.data_ptr(), _ptr(valid), current_stream_ptr()))
    return out, valid


# ------------------------------------------------------------------------------------ host-buffer path
def period_runstat_host(x_host, poff, op_code, thr, reducer_code, window, cmp_f64=False, want_valid=True,
                        workspace=None, out_host=None, valid_host=None):
    """End-to-end call with HOST buffers (the `_host` C-ABI entry point): ``x_host`` is a (T, C)
    float32 CPU tensor (ideally pinned); slabs are streamed H2D inside the call, results land in
    host memory.  Returns ``(out_host, valid_host, workspace)`` so that buffers can be reused."""
    _require_cuda()
    assert x_host.dtype == torch.float32 and x_host.is_contiguous() and not x_host.is_cuda
    T, C = x_host.shape
    P = len(poff) - 1
    poff_h = np.ascontiguousarray(np.asarray(poff, dtype=np.int32))
    lib = load()
    need = int(lib.xc_host_stream_workspace_bytes(T, C, poff_h.ctypes.data, P))
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device="cuda")
    if out_host is None:
        out_host = torch.empty((P, C), dtype=torch.float32).pin_memory()
    if want_valid and valid_host is None:
        valid_host = torch.empty((P, C), dtype=torch.int32).pin_memory()
    # the entry point works on its own non-blocking streams: nothing queued on torch's stream may still be
    # using a block the caching allocator has just recycled into `workspace`
    torch.cuda.current_stream().synchronize()
    check(lib.xc_period_runstat_f32_host(x_host.data_ptr(), T, C, poff_h.ctypes.data, P, op_code, float(thr),
                                         int(bool(cmp_f64)), reducer_code, int(window), out_host.data_ptr(),
                                         valid_host.data_ptr() if want_valid else None, workspace.data_ptr(),
                                         workspace.numel()))
    return out_host, (valid_host if want_valid else None), workspace


def bootstrap_doy_count(x2d, base_start, n_base_years, year_len, step_period, P, window, percentile, alpha, beta,
                        op_code):
    """(P, C) float64 bootstrapped exceedance counts for the in-base periods (0 elsewhere)."""
    T, C = x2d.shape
    sp = dev_ints(step_period, np.int32, x2d.device)
    assert sp.numel() == n_base_years * year_len
    scratch = torch.empty((P, C), dtype=torch.int32, device=x2d.device)
    out = torch.empty((P, C), dtype=torch.float64, device=x2d.device)
    check(load().xc_bootstrap_doy_count_f32(x2d.data_ptr(), T, C, x2d.stride(0), int(base_start), int(n_base_years),
                                            int(year_len), sp.data_ptr(), P, int(window), float(percentile),
                                            float(alpha), float(beta), op_code, scratch.data_ptr(), out.data_ptr(),
                                            current_stream_ptr()))
    return out


# ------------------------------------------------------------------------------------ rolling / spells
def rolling_period_reduce(x2d, poff, window, window_stat_code, center, stat_code):
    T, C = x2d.shape
    P = len(poff) - 1
    poff_d = dev_ints(poff, np.int32, x2d.device)
    out = torch.empty((P, C), dtype=torch.float32, device=x2d.device)
    check(load().xc_rolling_period_reduce_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(), P, int(window),
                                              window_stat_code, int(bool(center)), stat_code, out.data_ptr(),
                                              current_stream_ptr()))
    return out


def rolling_period_reduce_sel(x2d, poff, window, window_stat_code, center, stat_code, keep):
    """rolling_period_reduce with ``select_time`` on the rolled series (labels with keep[t] == 0 dropped)."""
    T, C = x2d.shape
    P = len(poff) - 1
    poff_d = dev_ints(poff, np.int32, x2d.device)
    k = dev_ints(np.asarray(keep, dtype=np.uint8), np.uint8, x2d.device)
    out = torch.empty((P, C), dtype=torch.float32, device=x2d.device)
    check(load().xc_rolling_period_reduce_sel_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(), P,
                                                  int(window), window_stat_code, int(bool(center)), stat_code,
                                                  k.data_ptr(), out.data_ptr(), current_stream_ptr()))
    return out


def spell_runstat(x2d, poff, window, window_stat_code, op_code, thr, reducer_code, resample_before_rl=True):
    T, C = x2d.shape
    P = len(poff) - 1
    poff_d = dev_ints(poff, np.int32, x2d.device)
    out = torch.empty((P, C), dtype=torch.float32, device=x2d.device)
    check(load().xc_spell_runstat_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(), P, int(window),
                                      window_stat_code, op_code, float(thr), reducer_code,
                                      int(bool(resample_before_rl)), out.data_ptr(), current_stream_ptr()))
    return out


def spell_mask(x2d, window, window_stat_code, op_code, thr, keep=None, drop_nan_adjacent=False):
    """(T, C) float32 spell mask with ``select_time`` applied (NaN out of season), see xc_spell_mask_f32."""
    T, C = x2d.shape
    k = None if keep is None else dev_ints(np.asarray(keep, dtype=np.uint8), np.uint8, x2d.device)
    out = torch.empty((T, C), dtype=torch.float32, device=x2d.device)
    check(load().xc_spell_mask_f32(x2d.data_ptr(), T, C, x2d.stride(0), int(window), window_stat_code, op_code,
                                   float(thr), _ptr(k), int(bool(drop_nan_adjacent)), out.data_ptr(),
                                   current_stream_ptr()))
    return out


# ------------------------------------------------------------------------------------ quantile mapping
def eqm_train(ref2d, hist2d, nq, kind_code):
    T, C = ref2d.shape
    assert hist2d.shape == ref2d.shape and ref2d.stride(0) == hist2d.stride(0)
    af = torch.empty((nq, C), dtype=torch.float32, device=ref2d.device)
    hq = torch.empty((nq, C), dtype=torch.float32, device=ref2d.device)
    lib = load()
    ws = torch.empty(int(lib.xc_eqm_train_workspace_bytes(T, C, int(nq))), dtype=torch.uint8, device=ref2d.device)
    check(lib.xc_eqm_train_f32(ref2d.data_ptr(), hist2d.data_ptr(), T, C, ref2d.stride(0), int(nq), kind_code,
                               af.data_ptr(), hq.data_ptr(), ws.data_ptr(), ws.numel(), current_stream_ptr()))
    return af, hq


def eqm_adjust(sim2d, af, hq, kind_code, interp_code):
    T, C = sim2d.shape
    scen = torch.empty((T, C), dtype=torch.float32, device=sim2d.device)
    check(load().xc_eqm_adjust_f32(sim2d.data_ptr(), T, C, sim2d.stride(0), af.data_ptr(), hq.data_ptr(),
                                   af.shape[0], kind_code, interp_code, scen.data_ptr(), current_stream_ptr()))
    return scen


#: upper bound of the QDM ranking scratch; larger grids are ranked in chunks of cells (6 T + 16 bytes per cell)
QDM_WORKSPACE_CAP = 2 << 30


def qdm_adjust(sim2d, af, nodes, kind_code, interp_code, want_sim_q=False, workspace_bytes=None):
    """Quantile delta mapping adjust (xc_qdm_adjust_f32): ``scen`` (T, C) float32 and, with ``want_sim_q``, the
    float64 percentage ranks ``sim_q`` (else None).  ``nodes``: the nq float32 quantile nodes of ``af`` (nq, C).
    ``workspace_bytes`` (default: all cells at once, capped by QDM_WORKSPACE_CAP; the smallest workspace when that
    does not fit) sets the ranking scratch, hence the number of cell chunks."""
    T, C = sim2d.shape
    nq = af.shape[0]
    assert af.shape == (nq, C) and af.is_contiguous() and af.dtype == torch.float32
    lib = load()
    if workspace_bytes is None:
        try:
            ws = torch.empty(min(int(lib.xc_qdm_adjust_workspace_bytes(T, C)), QDM_WORKSPACE_CAP), dtype=torch.uint8,
                             device=sim2d.device)
        except torch.cuda.OutOfMemoryError:
            ws = torch.empty(int(lib.xc_qdm_adjust_workspace_bytes(T, 32)), dtype=torch.uint8, device=sim2d.device)
    else:
        ws = torch.empty(int(workspace_bytes), dtype=torch.uint8, device=sim2d.device)
    nodes_d = torch.as_tensor(np.asarray(nodes, dtype=np.float32)).to(sim2d.device)
    scen = torch.empty((T, C), dtype=torch.float32, device=sim2d.device)
    sim_q = torch.empty((T, C), dtype=torch.float64, device=sim2d.device) if want_sim_q else None
    check(lib.xc_qdm_adjust_f32(sim2d.data_ptr(), T, C, sim2d.stride(0), af.data_ptr(), nodes_d.data_ptr(), nq,
                                kind_code, interp_code, scen.data_ptr(), _ptr(sim_q), ws.data_ptr(), ws.numel(),
                                current_stream_ptr()))
    return scen, sim_q


def dqm_train(ref2d, hist2d, nq, kind_code):
    """Detrended quantile mapping train (xc_dqm_train_f32): ``(af, hist_q, scaling)``, af / hist_q (nq, C) and
    scaling (C,) float32 -- EQM's quantiles of the mean-normalised ref and hist, and the ratio of their means."""
    T, C = ref2d.shape
    assert hist2d.shape == ref2d.shape and ref2d.stride(0) == hist2d.stride(0)
    af = torch.empty((nq, C), dtype=torch.float32, device=ref2d.device)
    hq = torch.empty((nq, C), dtype=torch.float32, device=ref2d.device)
    scaling = torch.empty(C, dtype=torch.float32, device=ref2d.device)
    lib = load()
    ws = torch.empty(int(lib.xc_dqm_train_workspace_bytes(T, C, int(nq))), dtype=torch.uint8, device=ref2d.device)
    check(lib.xc_dqm_train_f32(ref2d.data_ptr(), hist2d.data_ptr(), T, C, ref2d.stride(0), int(nq), kind_code,
                               af.data_ptr(), hq.data_ptr(), scaling.data_ptr(), ws.data_ptr(), ws.numel(),
                               current_stream_ptr()))
    return af, hq, scaling


def poly_fit(x2d, degree, kind_code=0, scaling=None):
    """Per-cell least-squares polynomial of ``degree`` over the valid steps (xc_poly_fit_f32): (degree + 1, C)
    float64 coefficients in the basis u_t = (2t - (T - 1)) / max(T - 1, 1).  With ``scaling`` ((C,) float32) the
    series fitted is float32(x + scaling) (kind 0) or float32(x * scaling) (kind 1)."""
    T, C = x2d.shape
    coef = torch.empty((int(degree) + 1, C), dtype=torch.float64, device=x2d.device)
    if scaling is not None:
        assert scaling.dtype == torch.float32 and scaling.is_contiguous() and scaling.numel() == C
    check(load().xc_poly_fit_f32(x2d.data_ptr(), T, C, x2d.stride(0), int(degree), kind_code, _ptr(scaling),
                                 coef.data_ptr(), current_stream_ptr()))
    return coef


def dqm_adjust(sim2d, af, hq, scaling, kind_code, interp_code, degree, want_coef=False):
    """Detrended quantile mapping adjust: the trend of float32(sim (+|*) scaling) (poly_fit), then one streaming pass
    (xc_dqm_adjust_f32).  Returns ``scen`` (T, C) float32, or ``(scen, coef)`` with ``want_coef``."""
    T, C = sim2d.shape
    nq = af.shape[0]
    for t in (af, hq):
        assert t.shape == (nq, C) and t.is_contiguous() and t.dtype == torch.float32
    coef = poly_fit(sim2d, degree, kind_code, scaling)
    scen = torch.empty((T, C), dtype=torch.float32, device=sim2d.device)
    check(load().xc_dqm_adjust_f32(sim2d.data_ptr(), T, C, sim2d.stride(0), af.data_ptr(), hq.data_ptr(),
                                   scaling.data_ptr(), coef.data_ptr(), nq, kind_code, interp_code, int(degree),
                                   scen.data_ptr(), current_stream_ptr()))
    return (scen, coef) if want_coef else scen


def detrend(x2d, degree):
    """``x - trend`` in float64 (T, C), the trend being the degree-``degree`` least-squares polynomial of x itself
    over its valid steps (poly_fit, then xc_detrend_apply_f32)."""
    T, C = x2d.shape
    coef = poly_fit(x2d, degree)
    out = torch.empty((T, C), dtype=torch.float64, device=x2d.device)
    check(load().xc_detrend_apply_f32(x2d.data_ptr(), T, C, x2d.stride(0), coef.data_ptr(), int(degree),
                                      out.data_ptr(), current_stream_ptr()))
    return out


def period_boundary_run(x2d, poff, op_code, thr, window, last=False, cmp_f64=False):
    """Index of the first (last) run of >= window steps per period, NaN if none (run_length.py:543-740)."""
    T, C = x2d.shape
    P = len(poff) - 1
    poff_d = dev_ints(poff, np.int32, x2d.device)
    out = torch.empty((P, C), dtype=torch.float32, device=x2d.device)
    check(load().xc_period_boundary_run_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(), P, op_code,
                                            float(thr), int(bool(cmp_f64)), int(window), int(bool(last)),
                                            out.data_ptr(), current_stream_ptr()))
    return out


def period_run_maxsum(x2d, poff, op_code, thr, window, resample_before_rl=True):
    """windowed_max_run_sum of the excess over ``thr`` per period (run_length.py:491-540)."""
    T, C = x2d.shape
    P = len(poff) - 1
    poff_d = dev_ints(poff, np.int32, x2d.device)
    out = torch.empty((P, C), dtype=torch.float32, device=x2d.device)
    check(load().xc_period_run_maxsum_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(), P, op_code,
                                          float(thr), int(window), int(bool(resample_before_rl)), out.data_ptr(),
                                          current_stream_ptr()))
    return out


def period_boundary_run_range(x2d, poff, range_lo, range_hi, op_code, thr, window, last=False, negate=False,
                              cell_lo=None, cmp_f64=False):
    """First/last run confined to [range_lo[p], range_hi[p]) of every period (run_length.py:1148-1331)."""
    T, C = x2d.shape
    P = len(poff) - 1
    poff_d = dev_ints(poff, np.int32, x2d.device)
    lo_d = dev_ints(range_lo, np.int32, x2d.device)
    hi_d = dev_ints(range_hi, np.int32, x2d.device)
    out = torch.empty((P, C), dtype=torch.float32, device=x2d.device)
    check(load().xc_period_boundary_run_range_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(),
                                                  lo_d.data_ptr(), hi_d.data_ptr(), P, op_code, float(thr),
                                                  int(bool(cmp_f64)), int(bool(negate)), int(window), int(bool(last)),
                                                  _ptr(cell_lo), out.data_ptr(), current_stream_ptr()))
    return out


def period_runstat2(x1, x2, poff, op1, thr1, op2, thr2, reducer_code, window, resample_before_rl=True, var_any=False):
    """Run statistics of (x1 op1 thr1) AND|OR (x2 op2 thr2) per period (heat_wave_* family)."""
    T, C = x1.shape
    assert x2.shape == x1.shape and x1.stride(0) == x2.stride(0)
    P = len(poff) - 1
    poff_d = dev_ints(poff, np.int32, x1.device)
    out = torch.empty((P, C), dtype=torch.float32, device=x1.device)
    check(load().xc_period_runstat2_f32(x1.data_ptr(), x2.data_ptr(), T, C, x1.stride(0), poff_d.data_ptr(), P, op1,
                                        float(thr1), op2, float(thr2), int(bool(var_any)), reducer_code, int(window),
                                        int(bool(resample_before_rl)), out.data_ptr(), current_stream_ptr()))
    return out


def mask_steps(x2d, keep):
    """``select_time`` with drop=False: NaN on the steps where ``keep`` is False (a new buffer)."""
    T, C = x2d.shape
    k = dev_ints(np.asarray(keep, dtype=np.uint8), np.uint8, x2d.device)
    out = torch.empty((T, C), dtype=torch.float32, device=x2d.device)
    check(load().xc_mask_steps_f32(x2d.data_ptr(), T, C, x2d.stride(0), k.data_ptr(), out.data_ptr(),
                                   current_stream_ptr()))
    return out


def period_runstat_gap(x2d, poff, op_code, thr, reducer_code, min_gap, window=1, cmp_f64=False):
    """Run statistics per period of the mask with holes < min_gap filled (generic.spell_mask(min_gap))."""
    T, C = x2d.shape
    P = len(poff) - 1
    poff_d = dev_ints(poff, np.int32, x2d.device)
    out = torch.empty((P, C), dtype=torch.float32, device=x2d.device)
    check(load().xc_period_runstat_gap_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(), P, op_code,
                                           float(thr), int(bool(cmp_f64)), reducer_code, int(window), int(min_gap),
                                           out.data_ptr(), current_stream_ptr()))
    return out


def period_run_quantile(x2d, poff, op_code, thr, q, window, resample_before_rl=True, cmp_f64=False):
    """Linear quantile ``q`` of the run lengths >= window per period (rle_statistics reducer "qNN")."""
    T, C = x2d.shape
    P = len(poff) - 1
    poff_h = np.ascontiguousarray(np.asarray(poff, dtype=np.int32))
    poff_d = dev_ints(poff_h, np.int32, x2d.device)
    out = torch.empty((P, C), dtype=torch.float32, device=x2d.device)
    check(load().xc_period_run_quantile_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(),
                                            poff_h.ctypes.data, P, op_code, float(thr), int(bool(cmp_f64)), float(q),
                                            int(window), int(bool(resample_before_rl)), out.data_ptr(),
                                            current_stream_ptr()))
    return out


# ------------------------------------------------------------------------------------ fused multi-output pass
def normalise_condition(op_code, thr):
    """(sgn, thr') with  x op thr  <=>  sgn * x > thr'  for every float32 x (NaN: False on both sides).
    ``thr`` is compared in float32 (numpy >= 2 weak-scalar rule, indices/generic.py:301-326).  Raises
    NotImplementedError for the conditions no strict ``>`` expresses: ``x >= -inf`` and ``x <= +inf`` (true for
    every non-NaN x, including the infinity itself, which has no float32 predecessor)."""
    gt, lt, ge, le = _lib.OPS[">"], _lib.OPS["<"], _lib.OPS[">="], _lib.OPS["<="]
    with np.errstate(over="ignore"):       # Python floats beyond float32 round to +-inf, as numpy compares them
        t = np.float32(thr)
        if op_code == gt:
            return 1.0, float(t)
        if op_code == lt:
            return -1.0, float(-t)
        if (op_code == ge and t == -np.inf) or (op_code == le and t == np.inf):
            raise NotImplementedError(f"the fused pass cannot express x {'>=' if op_code == ge else '<='} {float(t)}")
        if op_code == ge:                  # x >= t  <=>  x > pred(t)
            return 1.0, float(np.nextafter(t, np.float32(-np.inf)))
        if op_code == le:                  # x <= t  <=>  -x >= -t  <=>  -x > pred(-t)
            return -1.0, float(np.nextafter(np.float32(-t), np.float32(-np.inf)))
    raise NotImplementedError("the fused pass takes the operators >, >=, <, <=")


def period_multi(x2d, poff, plan, n_slots):
    """One streaming pass producing every output of ``plan`` (a ``_lib.MultiPlan``); returns the
    ``(n_slots, P, C)`` float32 slot buffer (count slots hold int32 bits: view them with ``.view(torch.int32)``).
    The kernel reads four cells per 16-byte load; a grid whose cell count or row stride is not a multiple of 4
    (small regional grids) is copied once into a zero-padded buffer that is."""
    import ctypes
    T, C = x2d.shape
    P = len(poff) - 1
    if C % 4 or x2d.stride(0) % 4 or x2d.stride(1) != 1 or x2d.data_ptr() % 16:
        xp = torch.zeros((T, (C + 3) // 4 * 4), dtype=torch.float32, device=x2d.device)
        xp[:, :C] = x2d
        return period_multi(xp, poff, plan, n_slots)[:, :, :C].contiguous()
    poff_d = dev_ints(poff, np.int32, x2d.device)
    out = torch.empty((max(1, n_slots), P, C), dtype=torch.float32, device=x2d.device)
    check(load().xc_period_multi_f32(x2d.data_ptr(), T, C, x2d.stride(0), poff_d.data_ptr(), P, ctypes.byref(plan),
                                     out.data_ptr(), int(n_slots), current_stream_ptr()))
    return out


# ------------------------------------------------------------------------------------ standardized indices
def rolling_mean(x2d, window):
    """``rolling(time=window).mean(skipna=False)`` as a new (T, C) float32 series (xc_rolling_mean_f32)."""
    T, C = x2d.shape
    out = torch.empty((T, C), dtype=torch.float32, device=x2d.device)
    check(load().xc_rolling_mean_f32(x2d.data_ptr(), T, C, x2d.stride(0), int(window), out.data_ptr(), C,
                                     current_stream_ptr()))
    return out


def si_fit(x2d, group_offsets, steps, dist_code, method_code, zero_inflated, floc):
    """Fit every (group, cell) sample (xc_si_fit_f32).  ``group_offsets`` (G + 1) / ``steps``: host int arrays,
    the CSR of each group's calibration steps.  Returns ``(params (G, 3, C) float64, n_zeros, n_notnull (G, C)
    int32 or None, status int)``; reading the status synchronises the stream."""
    T, C = x2d.shape
    goff = np.ascontiguousarray(np.asarray(group_offsets, dtype=np.int32))
    G = goff.size - 1
    max_n = int(np.diff(goff).max()) if G > 0 else 0
    st = np.ascontiguousarray(np.asarray(steps, dtype=np.int32))
    goff_d = dev_ints(goff, np.int32, x2d.device)
    steps_d = dev_ints(st if st.size else np.zeros(1, np.int32), np.int32, x2d.device)
    lib = load()
    ws = torch.empty(int(lib.xc_si_fit_workspace_bytes(C, max_n)), dtype=torch.uint8, device=x2d.device)
    params = torch.empty((G, 3, C), dtype=torch.float64, device=x2d.device)
    nz = torch.empty((G, C), dtype=torch.int32, device=x2d.device) if zero_inflated else None
    nn = torch.empty((G, C), dtype=torch.int32, device=x2d.device) if zero_inflated else None
    status = torch.zeros(1, dtype=torch.int32, device=x2d.device)
    check(lib.xc_si_fit_f32(x2d.data_ptr(), T, C, x2d.stride(0), goff_d.data_ptr(), steps_d.data_ptr(), G, max_n,
                            int(dist_code), int(method_code), int(bool(zero_inflated)), float(floc), params.data_ptr(),
                            _ptr(nz), _ptr(nn), status.data_ptr(), ws.data_ptr(), ws.numel(), current_stream_ptr()))
    return params, nz, nn, int(status.item())


def si_apply(x2d, group_of_step, params, n_zeros, n_notnull, dist_code, interp=1.0, alpha=0.0, beta=1.0):
    """(T, C) float64 standardized index (xc_si_apply_f32); ``group_of_step`` host int array, -1 = NaN;
    ``n_zeros`` / ``n_notnull`` None for a distribution without zero inflation."""
    T, C = x2d.shape
    G = params.shape[0]
    assert params.shape == (G, 3, C) and params.dtype == torch.float64 and params.is_contiguous()
    zi = n_zeros is not None
    if zi:
        for t in (n_zeros, n_notnull):
            assert t.shape == (G, C) and t.dtype == torch.int32 and t.is_contiguous()
    gos = dev_ints(np.asarray(group_of_step, dtype=np.int16), np.int16, x2d.device)
    out = torch.empty((T, C), dtype=torch.float64, device=x2d.device)
    check(load().xc_si_apply_f32(x2d.data_ptr(), T, C, x2d.stride(0), gos.data_ptr(), G, params.data_ptr(),
                                 _ptr(n_zeros), _ptr(n_notnull), int(dist_code), int(zi), float(interp), float(alpha),
                                 float(beta), out.data_ptr(), C, current_stream_ptr()))
    return out


# ------------------------------------------------------------------------------------ frequency analysis
def ev_fit(x2d, dist_code):
    """Fit every column of the (T, C) float32 series (xc_ev_fit_f32).  Returns ``(params (2 | 3, C) float64,
    status int)``; reading the status synchronises the stream."""
    T, C = x2d.shape
    lib = load()
    ws = torch.empty(int(lib.xc_ev_fit_workspace_bytes(T, C)), dtype=torch.uint8, device=x2d.device)
    params = torch.empty((3 if dist_code == _lib.EV_DISTS["genextreme"] else 2, C), dtype=torch.float64,
                         device=x2d.device)
    status = torch.zeros(1, dtype=torch.int32, device=x2d.device)
    check(lib.xc_ev_fit_f32(x2d.data_ptr(), T, C, x2d.stride(0), int(dist_code), params.data_ptr(),
                            status.data_ptr(), ws.data_ptr(), ws.numel(), current_stream_ptr()))
    return params, int(status.item())


def ev_transform(params, dist_code, kind_code, q):
    """(nq, C) float64 ppf / isf / cdf of the fitted laws (xc_ev_transform_f64); ``params`` (2 | 3, C) float64
    tensor (copied to the device when it is not there), ``q`` host probabilities or values."""
    P, C = params.shape
    if not params.is_cuda:
        _require_cuda()
        params = params.to("cuda")
    params = params.to(torch.float64).contiguous()
    qd = torch.as_tensor(np.ascontiguousarray(q, dtype=np.float64).ravel()).to(params.device)
    out = torch.empty((qd.numel(), C), dtype=torch.float64, device=params.device)
    check(load().xc_ev_transform_f64(params.data_ptr(), C, int(dist_code), int(kind_code), qd.data_ptr(),
                                     qd.numel(), out.data_ptr(), current_stream_ptr()))
    return out


# ------------------------------------------------------------------------------------ spatial analogues
def analog(target, cand, method_code, param, consts):
    """(K, C) float64 dissimilarities (xc_analog_f32) of the (K, n, d) float32 targets against the (m, d, C) float32
    candidates (unit cell stride; a row stride > C works in place), with ``consts`` the (K, d | d * d) float64
    per-target constants or None.  Returns ``(out, status)``; reading the status synchronises the stream."""
    K, n, d = target.shape
    m, _, C = cand.shape
    assert target.dtype == torch.float32 and target.is_contiguous()
    assert cand.dtype == torch.float32 and cand.stride(2) == 1 and cand.stride(0) == d * cand.stride(1)
    out = torch.empty((K, C), dtype=torch.float64, device=cand.device)
    status = torch.zeros(1, dtype=torch.int32, device=cand.device)
    check(load().xc_analog_f32(target.data_ptr(), n, K, cand.data_ptr(), m, C, cand.stride(1), d, int(method_code),
                               float(param), _ptr(consts), out.data_ptr(), status.data_ptr(), current_stream_ptr()))
    return out, int(status.item())


# ------------------------------------------------------------------------------------ evapotranspiration
def _pet_inputs(inputs):
    """Host array of the XC_PET_N_IN input pointers and (T, C, ld) of the (T, C) float32 device series."""
    import ctypes
    ref = next(x for x in inputs if x is not None)
    T, C = ref.shape
    ld = ref.stride(0)
    for x in inputs:
        if x is not None and (tuple(x.shape) != (T, C) or x.stride(0) != ld or x.stride(1) != 1
                              or x.dtype != torch.float32):
            raise ValueError("pet: the inputs must share their (T, C) float32 layout")
    return (ctypes.c_void_p * len(inputs))(*[_ptr(x) for x in inputs]), T, C, ld, ref.device


def pet_daily(inputs, table, lat_index, params):
    """PET or the water budget of a daily method (xc_pet_daily_f32): ``inputs`` the XC_PET_N_IN (T, C) float32
    device series or None (a row stride > C works in place), ``table`` (T, L) float64 and ``lat_index`` (C,) int32
    device tensors (None for allen98), ``params`` a ``_lib.PetParams``.  Returns (T, C) float32 with the row stride
    of the inputs."""
    import ctypes
    ptrs, T, C, ld, dev = _pet_inputs(inputs)
    out = torch.empty((T, ld), dtype=torch.float32, device=dev)[:, :C]
    L = 0 if table is None else table.shape[1]
    check(load().xc_pet_daily_f32(ptrs, T, C, ld, _ptr(table), L, _ptr(lat_index), ctypes.byref(params),
                                  out.data_ptr(), current_stream_ptr()))
    return out


def pet_monthly(inputs, moff, yoff, mdays, table, lat_index, params):
    """PET or the water budget of a monthly method (xc_pet_monthly_f32) from daily series: ``moff`` (M + 1) and
    ``yoff`` (Y + 1) int32 host arrays, ``mdays`` (M,) float64 host array, ``table`` (M, L) float64 and
    ``lat_index`` (C,) int32 device tensors.  Returns (M, C) float32."""
    import ctypes
    ptrs, T, C, ld, dev = _pet_inputs(inputs)
    moff_d, yoff_d = dev_ints(moff, np.int32, dev), dev_ints(yoff, np.int32, dev)
    mdays_d = torch.from_numpy(np.ascontiguousarray(mdays, dtype=np.float64)).to(dev)
    M = moff_d.numel() - 1
    out = torch.empty((M, C), dtype=torch.float32, device=dev)
    check(load().xc_pet_monthly_f32(ptrs, T, C, ld, moff_d.data_ptr(), M, yoff_d.data_ptr(), yoff_d.numel() - 1,
                                    mdays_d.data_ptr(), table.data_ptr(), table.shape[1], lat_index.data_ptr(),
                                    ctypes.byref(params), out.data_ptr(), current_stream_ptr()))
    return out


# ------------------------------------------------------------------------------------ ensembles
def ens_percentiles(x2d, percentiles, alpha, beta, min_members):
    """Percentiles along the member axis of an (R, N) float32 matrix (xc_ens_percentiles_f32; column views with
    a row stride > N work in place).  Returns (n_per, N): float64 for R >= 2, float32 for R == 1."""
    R, N = x2d.shape
    assert x2d.dtype == torch.float32 and x2d.stride(1) == 1
    per = np.ascontiguousarray(np.asarray(percentiles, dtype=np.float64).ravel())
    out = torch.empty((per.size, N), dtype=torch.float64 if R >= 2 else torch.float32, device=x2d.device)
    for p0 in range(0, per.size, _lib.ENS_MAX_PER):
        chunk = per[p0:p0 + _lib.ENS_MAX_PER]
        check(load().xc_ens_percentiles_f32(x2d.data_ptr(), R, N, x2d.stride(0), chunk.ctypes.data, chunk.size,
                                            float(alpha), float(beta), int(min_members), out[p0].data_ptr(),
                                            current_stream_ptr()))
    return out


def ens_moments(x2d, weights, min_members):
    """(mean, std, min, max) along the member axis of an (R, N) float32 matrix (xc_ens_moments_f32): mean / std
    float32 without weights, float64 with ``weights`` (a float64 device tensor of R values)."""
    R, N = x2d.shape
    assert x2d.dtype == torch.float32 and x2d.stride(1) == 1
    dt = torch.float32 if weights is None else torch.float64
    mean, std = (torch.empty(N, dtype=dt, device=x2d.device) for _ in range(2))
    vmin, vmax = (torch.empty(N, dtype=torch.float32, device=x2d.device) for _ in range(2))
    check(load().xc_ens_moments_f32(x2d.data_ptr(), R, N, x2d.stride(0), _ptr(weights), int(min_members),
                                    mean.data_ptr(), std.data_ptr(), vmin.data_ptr(), vmax.data_ptr(),
                                    current_stream_ptr()))
    return mean, std, vmin, vmax


def ens_robustness(fut, ref, weights, test_code, param, strict_sign, want_pvals, ref_annual=None, ys_time=None):
    """Robustness fractions (7, C) float64 and the (R, C) float32 p-values (or None) of ``fut`` / ``ref`` given as
    (R, T, C) float32 device tensors with unit cell stride (``ref`` None: ``fut`` is (R, 1, C) deltas).  ipcc-ar6-c
    also takes ``ref_annual`` (R, P, C) float32 (the YS means of ``ref``) and ``ys_time`` (P) float64 device
    tensors."""
    R, Tf, C = fut.shape
    assert fut.dtype == torch.float32 and fut.stride(2) == 1
    if ref is not None:
        assert ref.dtype == torch.float32 and ref.stride(2) == 1 and ref.shape[0] == R and ref.shape[2] == C
    frac = torch.empty((7, C), dtype=torch.float64, device=fut.device)
    pvals = torch.empty((R, C), dtype=torch.float32, device=fut.device) if want_pvals else None
    Tr, sr_r, sr_t = (ref.shape[1], ref.stride(0), ref.stride(1)) if ref is not None else (0, 0, 0)
    P, sa_r = 0, 0
    if ref_annual is not None:
        assert ref_annual.dtype == torch.float32 and ref_annual.stride(2) == 1 and ref_annual.stride(1) == C
        assert ys_time.dtype == torch.float64 and ys_time.is_contiguous() and ys_time.numel() == ref_annual.shape[1]
        P, sa_r = ref_annual.shape[1], ref_annual.stride(0)
    check(load().xc_ens_robustness_f32(fut.data_ptr(), Tf, fut.stride(0), fut.stride(1), _ptr(ref), Tr, sr_r, sr_t,
                                       _ptr(ref_annual), P, sa_r, _ptr(ys_time), R, C, _ptr(weights), int(test_code), float(param), int(bool(strict_sign)),
                                       frac.data_ptr(), _ptr(pvals), current_stream_ptr()))
    return frac, pvals


# ------------------------------------------------------------------------------------ fire weather
FWI_OUTPUTS = ("DC", "DMC", "FFMC", "ISI", "BUI", "FWI", "DSR")


def fwi_params(season_method=None, overwintering=False, dry_start=None, initial_start_up=True, in_affine=None, **p):
    """``_lib.FwiParams`` from the keyword parameters of ``fire_weather_ufunc`` (indices/fire/_cffwis.py:161-178:
    thresholds compare in float32 with the float32 data, as numpy does for Python scalars)."""
    P = _lib.FwiParams()
    P.season_mode = _lib.FWI_SEASONS[season_method]
    P.dry_start = _lib.FWI_DRY_STARTS[dry_start]
    P.overwintering, P.initial_start_up = int(bool(overwintering)), int(bool(initial_start_up))
    for k in ("temp_condition_days", "snow_condition_days", "snow_cover_days"):
        setattr(P, k, int(p[k]))
    for k in ("temp_start_thresh", "temp_end_thresh", "snow_thresh", "prec_thresh", "snow_min_mean_depth", "dc_start",
              "dmc_start", "ffmc_start", "dc_dry_factor", "dmc_dry_factor", "snow_min_cover_frac", "carry_over_fraction",
              "wetting_efficiency_fraction"):
        setattr(P, k, float(p[k]))
    P.min_dc = float(p["dc_start"])
    for i, (scale, offset) in enumerate(in_affine or [(1.0, 0.0)] * 5):   # tas, pr, hurs, ws, snd
        P.in_scale[i], P.in_offset[i] = scale, offset
    return P


def fire_weather(tas, pr, hurs, ws, snd, month, lat, season_mask, dc0, dmc0, ffmc0, winter_pr, outputs, params):
    """The fire-weather day loop on ``(T, C)`` float32 device series (``xc_fwi_f32``).

    ``month`` int8[T] host array, ``lat`` float64[C] host array or device tensor; ``season_mask`` (T, C) uint8 / previous codes (C,)
    float32 device tensors or None.  ``outputs``: names among DC..DSR, "season_mask", "winter_pr".
    Returns a dict name -> device tensor.
    """
    import ctypes
    ref = tas if tas is not None else pr
    T, C = ref.shape
    dev = ref.device
    ld = ref.stride(0)
    for x in (tas, pr, hurs, ws, snd):
        if x is not None and (tuple(x.shape) != (T, C) or x.stride(0) != ld or x.dtype != torch.float32):
            raise ValueError("fire_weather: the inputs must share their (T, C) float32 layout")
    if season_mask is not None and (tuple(season_mask.shape) != (T, C) or season_mask.dtype != torch.uint8
                                    or season_mask.stride(0) != ld):
        raise ValueError("fire_weather: season_mask must be (T, C) uint8 with the layout of the inputs")
    month_d = dev_ints(np.asarray(month, dtype=np.int8), np.int8, dev)
    if lat is None or isinstance(lat, torch.Tensor):        # a float64 device tensor is used as it is
        lat_d = lat
    else:
        lat_d = torch.from_numpy(np.ascontiguousarray(lat, dtype=np.float64)).to(dev)
    if lat_d is not None and (lat_d.dtype != torch.float64 or lat_d.numel() != C):
        raise ValueError("fire_weather: lat must hold one float64 value per cell")
    out = {}
    for name in outputs:
        if name in FWI_OUTPUTS:      # outputs use the leading dimension of the inputs
            out[name] = torch.empty((T, ld), dtype=torch.float32, device=dev)[:, :C]
        elif name == "season_mask":
            out[name] = torch.empty((T, ld), dtype=torch.uint8, device=dev)[:, :C]
        elif name == "winter_pr":
            out[name] = torch.empty(C, dtype=torch.float32, device=dev)
        else:
            raise ValueError(f"unknown fire weather output {name!r}")
    optr = [_ptr(out.get(n)) for n in FWI_OUTPUTS]
    check(load().xc_fwi_f32(_ptr(tas), _ptr(pr), _ptr(hurs), _ptr(ws), _ptr(snd), _ptr(season_mask), month_d.data_ptr(),
                            _ptr(lat_d), _ptr(dc0), _ptr(dmc0), _ptr(ffmc0), _ptr(winter_pr), T, C, ld,
                            ctypes.byref(params), *optr, _ptr(out.get("season_mask")), _ptr(out.get("winter_pr")),
                            current_stream_ptr()))
    return out


def to_device_f32(values):
    """Any array (numpy, torch) as a float32 CUDA tensor of the same shape."""
    _require_cuda()
    if isinstance(values, torch.Tensor):
        return values.to(device="cuda", dtype=torch.float32)
    return torch.from_numpy(np.ascontiguousarray(np.asarray(values), dtype=np.float32)).to("cuda")


def fire_elementwise(kind, a, b=None, p=(0.0, 0.0, 0.0)):
    """One of the element-wise fire-weather functions on float32 device tensors (``xc_fwi_elementwise_f32``)."""
    if b is not None and tuple(b.shape) != tuple(a.shape):
        raise ValueError("fire_elementwise: the two inputs must share their shape")
    a = a.contiguous()
    b = None if b is None else b.contiguous()
    out = torch.empty_like(a)
    check(load().xc_fwi_elementwise_f32(_lib.FWI_ELEMENTWISE[kind], a.data_ptr(), _ptr(b), a.numel(), float(p[0]),
                                        float(p[1]), float(p[2]), out.data_ptr(), current_stream_ptr()))
    return out
