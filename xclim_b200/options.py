"""Package options, in the style of ``xclim.set_options`` (core/options.py).

``device_outputs`` (default False): functions called with a :class:`xclim_b200.Field` return their
result as a Field whose ``values`` is a CUDA tensor instead of copying it to the host, so that
a batch of indices over device-resident inputs runs without a device->host round trip per call
(``Field.numpy()`` materialises it).  xarray inputs always get numpy-backed DataArrays back.

``check_missing`` / ``missing_options`` (like xclim's options of the same names, core/options.py): the
missing-value criterion of the indicator-level entry points ``xclim_b200.atmos.*`` -- "any" (default),
"pct" (``{"tolerance": ...}``), "at_least_n" (``{"n": ...}``), "wmo" (``{"nm": ..., "nc": ...}``) or "skip".

``rle_nan_adjacent`` ("count", default | "drop"): spell statistics with a ``select_time`` indexer -- a spell that is
already under way on the first selected day counts with its in-season length (the reference's per-series path,
tests/test_indices.py:4116-4126) or is dropped (what its whole-array ``rle`` does next to a NaN, run_length.py:264).

``stream_min_bytes`` / ``stream_slab_bytes``: host-backed inputs at least this large are streamed through HBM
in lat slabs of about ``stream_slab_bytes`` (H2D of slab k+1 overlapped with the kernels of slab k).

``sdba_extra_output`` (default False): ``sdba.QuantileDeltaMapping.adjust`` returns ``{"scen": ..., "sim_q": ...}``
(``sim_q``: the float64 percentage ranks of ``sim``) instead of ``scen`` alone, like ``xsdba.set_options(
extra_output=True)``.
"""
from __future__ import annotations

OPTIONS = {"device_outputs": False, "rle_nan_adjacent": "count", "check_missing": "any", "missing_options": {},
           "sdba_extra_output": False,
           # end-to-end slab streaming of host inputs (xclim_b200/streaming.py): inputs smaller than
           # stream_min_bytes are unwrapped in one piece; one slab of one input is about stream_slab_bytes
           "stream_min_bytes": 256 << 20, "stream_slab_bytes": 1 << 30, "_in_stream": False}


class set_options:
    """``with set_options(device_outputs=True): ...`` or a plain call for a global change."""

    def __init__(self, **kwargs):
        self._old = {}
        for k, v in kwargs.items():
            if k not in OPTIONS:
                raise ValueError(f"argument name {k!r} is not in the set of valid options {set(OPTIONS)!r}")
            self._old[k] = OPTIONS[k]
            OPTIONS[k] = v

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        OPTIONS.update(self._old)
