"""Indicator-level entry points for the headline configurations: index + fused missing-value mask.

The reference's ``Indicator.__call__`` (core/indicator.py:865-944) runs ``compute`` and then, in
``CheckMissingIndicator._postprocess`` (:1522-1549), a SECOND full read of every input to build the
``MissingAny`` mask (core/missing.py:296-322).  Here the non-NaN step count per period comes out of the
same streaming kernel as the index (the ``valid_count`` output of the C ABI), so the mask costs no
extra pass.  Only the numeric part of the Indicator is mirrored: period values are NaN where a period
has a missing step, ``units`` follow the stock indicators (``days`` / input units); CF attribute
templating, cfchecks and translations stay with the real xclim (INTEGRATION.md).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, device
from .field import attrs_of
from .generic import _unwrap, _wrap_periods
from .options import OPTIONS, set_options
from .units import threshold_in_units_of


def _mask_missing(out, valid, poff, expected=None):
    """NaN where the period does not hold every step a complete period has (``expected``: TimeAxis.
    expected_period_lengths; the observed period lengths when not given)."""
    n = np.diff(poff) if expected is None else np.asarray(expected)
    n = torch.from_numpy(n.astype(np.int32)).to(out.device)[:, None]
    res = out.to(torch.float64) if out.dtype in (torch.int32, torch.int64) else out.clone()
    res[valid != n] = float("nan")
    return res


def maximum_consecutive_dry_days(pr, thresh="1 mm/day", freq="YS", resample_before_rl=True, **indexer):
    """``xclim.atmos.maximum_consecutive_dry_days`` (identifier ``cdd``, indicators/atmos/_precip.py:237-247):
    the index of indices/_threshold.py:2895-2937 with periods holding a missing day set to NaN."""
    if indexer or OPTIONS["check_missing"] != "any":
        # select_time on the input / another missing-value criterion: the generic wrapper (one extra pass)
        from . import indices
        return with_missing_any(indices.maximum_consecutive_dry_days)(pr, thresh=thresh, freq=freq,
                                                                      resample_before_rl=resample_before_rl, **indexer)
    thr = threshold_in_units_of(thresh, pr)
    x2d, cell_shape, other, ta = _unwrap(pr)
    poff = ta.period_offsets(freq)
    out, valid = device.period_runstat(x2d, poff, _lib.OPS["<"], thr, _lib.RL_REDUCERS["max"], 1, resample_before_rl,
                                       want_valid=True)
    attrs = attrs_of(pr)
    attrs.update(units="days", standard_name="number_of_days_with_lwe_thickness_of_precipitation_amount_below_threshold",
                 cell_methods="time: maximum over days")
    return _wrap_periods(pr, _mask_missing(out, valid, poff, ta.expected_period_lengths(freq)), cell_shape, other, ta, freq, attrs, dtype=np.float32,
                         name="cdd")


def tg_mean(tas, freq="YS", **indexer):
    """``xclim.atmos.tg_mean`` (indicators/atmos/_temperature.py:475-485)."""
    if indexer or OPTIONS["check_missing"] != "any":
        from . import indices
        return with_missing_any(indices.tg_mean)(tas, freq=freq, **indexer)
    x2d, cell_shape, other, ta = _unwrap(tas)
    poff = ta.period_offsets(freq)
    out, valid = device.period_reduce(x2d, poff, _lib.STATS["mean"], want_valid=True)
    attrs = attrs_of(tas)
    attrs.update(cell_methods="time: mean over days")
    return _wrap_periods(tas, _mask_missing(out, valid, poff, ta.expected_period_lengths(freq)), cell_shape, other, ta, freq, attrs, name="tg_mean")


def tx90p(tasmax, tasmax_per, freq="YS", bootstrap=False, op=">", **indexer):
    """``xclim.atmos.tx90p`` (indicators/atmos/_temperature.py:1269-1281): counts become float with NaN
    where the period has a missing day."""
    from .indices import tx90p as index_tx90p
    if indexer or OPTIONS["check_missing"] != "any":
        return with_missing_any(index_tx90p)(tasmax, tasmax_per, freq=freq, bootstrap=bootstrap, op=op, **indexer)
    if bootstrap:
        out = index_tx90p(tasmax, tasmax_per, freq=freq, bootstrap=True, op=op)
        x2d, cell_shape, other, ta = _unwrap(tasmax)
        poff = ta.period_offsets(freq)
        _, valid = device.period_count(x2d, poff, _lib.OP_NOTNAN, 0.0, want_valid=True)
        vals = out.values if hasattr(out.values, "is_cuda") else torch.from_numpy(np.asarray(out.values, np.float64))
        vals = vals.reshape(len(poff) - 1, -1).to(x2d.device)
        masked = _mask_missing(vals, valid, poff, ta.expected_period_lengths(freq))
        attrs = attrs_of(out)
        attrs["units"] = "days"
        return _wrap_periods(tasmax, masked, cell_shape, other, ta, freq, attrs, dtype=np.float64, name="tx90p")
    from .indices import _percentile_table_count
    code = _lib.op_code(op, (">", ">="))
    cnt, valid, (cell_shape, other, ta) = _percentile_table_count(tasmax, tasmax_per, code, freq, want_valid=True)
    attrs = attrs_of(tasmax)
    attrs.update(units="days", cell_methods="time: sum over days")
    masked = _mask_missing(cnt, valid, ta.period_offsets(freq), ta.expected_period_lengths(freq))
    return _wrap_periods(tasmax, masked, cell_shape, other, ta, freq, attrs, dtype=np.float64, name="tx90p")


# ---- generic indicator wrapper ---------------------------------------------------------------------------
def with_missing_any(index_fn, name=None):
    """Indicator-level version of an index function: the same call, then periods in which ANY input
    variable has a missing (NaN) step become NaN -- ``CheckMissingIndicator._postprocess``
    (core/indicator.py:1522-1549) with the default ``MissingAny`` (core/missing.py:310-322).  The
    non-NaN counts come from one extra streaming pass per input (``xc_period_count_f32`` with the
    NOTNAN operator); the three hand-written entry points above fuse that count into the index kernel."""
    import functools
    import inspect

    from .field import Field, dims_of, is_xarray

    sig = inspect.signature(index_fn)
    INDEXERS = ("season", "month", "doy_bounds", "date_bounds", "include_bounds")

    @functools.wraps(index_fn)
    def indicator(*args, **kwargs):
        # select_time indexers are an INDICATOR-level feature (ResamplingIndicatorWithIndexing,
        # core/indicator.py:1611-1673): the inputs are masked (NaN outside the selection) before the index runs
        indexer = {k: kwargs.pop(k) for k in INDEXERS if k in kwargs and k not in sig.parameters}
        bound = sig.bind(*args, **kwargs)
        bound.apply_defaults()
        freq = bound.arguments.get("freq")
        bad = None
        xr_template = None
        for key, val in list(bound.arguments.items()):
            if not (isinstance(val, Field) or is_xarray(val)) or "time" not in dims_of(val):
                continue                     # thresholds, percentile tables (dayofyear), options
            x2d, cell_shape, other, ta = _unwrap(val, indexer)
            if indexer:
                # the masked series stays in HBM as a Field; DataArray inputs get their result re-labelled below
                if is_xarray(val):
                    xr_template = val if xr_template is None else xr_template
                    coords = {d: np.asarray(val.coords[d].values) for d in other if d in val.coords}
                else:
                    coords = {k: v for k, v in val.coords.items() if k != "time"}
                bound.arguments[key] = Field(x2d.reshape((x2d.shape[0],) + cell_shape), ("time",) + other, ta, coords,
                                             dict(val.attrs), val.name)
            method = OPTIONS["check_missing"]
            if freq is None or method == "skip":
                continue
            poff = ta.period_offsets(freq)
            if method == "any":
                _, valid = device.period_count(x2d, poff, _lib.OP_NOTNAN, 0.0, want_valid=True)
                n = torch.from_numpy(ta.expected_period_lengths(freq, **indexer).astype(np.int32))
                miss = (valid != n.to(valid.device)[:, None]).reshape((len(poff) - 1,) + cell_shape)
            else:
                from . import missing as _missing
                fn = {"pct": _missing.missing_pct, "at_least_n": _missing.at_least_n_valid,
                      "wmo": _missing.missing_wmo}.get(method)
                if fn is None:
                    raise ValueError(f"unknown check_missing method {method!r}")
                masked_in = Field(x2d.reshape((x2d.shape[0],) + cell_shape), ("time",) + other, ta, {}, dict(val.attrs))
                mopts = OPTIONS["missing_options"]
                if isinstance(mopts.get(method), dict):      # xclim's nested form {"pct": {"tolerance": ...}}
                    mopts = mopts[method]
                with set_options(device_outputs=True):
                    m = fn(masked_in, freq, **mopts, **(indexer if method != "wmo" else {}))
                miss = m.values if hasattr(m.values, "is_cuda") else torch.from_numpy(np.asarray(m.values))
                miss = miss.to(x2d.device).reshape((len(poff) - 1,) + cell_shape).bool()
            bad = miss if bad is None else (bad | miss)
        out = index_fn(*bound.args, **bound.kwargs)
        if xr_template is not None:          # DataArray in -> DataArray out (the index ran on masked Fields)
            from .streaming import _assemble

            def relabel(o):
                if not isinstance(o, Field):
                    return o
                v = o.values
                return _assemble(xr_template, o, v.cpu().numpy() if hasattr(v, "is_cuda") else v, None)
            out = tuple(relabel(o) for o in out) if isinstance(out, tuple) else relabel(out)
        if bad is None:
            return out
        outs = out if isinstance(out, tuple) else (out,)
        masked = []
        for o in outs:
            v = o.values
            if hasattr(v, "is_cuda"):
                v = torch.where(bad.to(v.device), torch.full_like(v, float("nan"), dtype=torch.float64), v.to(torch.float64))
            else:
                v = np.where(bad.cpu().numpy(), np.nan, np.asarray(v, dtype=np.float64))
            if is_xarray(o):
                masked.append(o.copy(data=v))
            else:
                masked.append(Field(v, o.dims, o.time, dict(o.coords), dict(o.attrs), o.name))
        return tuple(masked) if isinstance(out, tuple) else masked[0]

    indicator.__name__ = name or index_fn.__name__
    from .streaming import streamed
    return streamed(indicator)       # host-backed inputs: missing counts + index per lat slab


from .chill import atmos_chill_portions as chill_portions, atmos_chill_units as chill_units  # noqa: E402,F401


def _stream_fused():
    from .streaming import streamed
    g = globals()
    for nm in ("maximum_consecutive_dry_days", "tg_mean", "tx90p"):
        g[nm] = streamed(g[nm])


_stream_fused()


def _register_batch():
    """``atmos.<name>`` for every index of the batch-of-50 list that has no hand-fused version above."""
    from . import indices
    g = globals()
    for nm, _var in indices.BATCH_INDICATORS:
        if nm not in g:
            g[nm] = with_missing_any(getattr(indices, nm), nm)


_register_batch()


def __getattr__(name):
    """Any other index of :mod:`xclim_b200.indices` at indicator level, built on first use."""
    from . import indices
    fn = getattr(indices, name, None)
    if callable(fn) and not name.startswith("_"):
        wrapped = with_missing_any(fn, name)
        globals()[name] = wrapped
        return wrapped
    raise AttributeError(f"module 'xclim_b200.atmos' has no attribute {name!r}")

