"""GPU tests of host-layer compositions: existing, verified kernels in new combinations."""
import numpy as np
import pytest

from oracle import xclim_oracle as O
from xb_helpers import make_field

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("win_reducer,op,thr", [("sum", "<", 1.0), ("min", ">=", 0.5), ("mean", ">", 2.0), ("max", "<", 3.0)])
@pytest.mark.parametrize("min_gap", [2, 4])
def test_spell_length_statistics_min_gap_with_window(cuda, win_reducer, op, thr, min_gap):
    """generic.spell_mask(window > 1, min_gap > 1) (indices/generic.py:519-538): the rolling-window mask
    (xc_spell_mask_f32) followed by the window-1 runs_with_holes kernel on it (xc_period_runstat_gap_f32)."""
    from xclim_b200 import generic
    rng = np.random.default_rng(45)
    x = rng.gamma(0.4, 6.0, size=(365 * 2 + 17, 3, 7)).astype(np.float32)
    x[rng.random(x.shape) < 0.45] = 0
    x = (np.round(x * 4) / 4).astype(np.float32)      # window sums exact in any order (as the verified window tests)
    x[rng.random(x.shape) < 0.003] = np.nan
    da = make_field(x, "2001-01-01", units="mm/d")
    for freq in ("YS", "MS"):
        poff = da.time.period_offsets(freq)
        got = generic.spell_length_statistics(da, thr, 3, win_reducer, op, ["max", "sum", "count"], freq, min_gap=min_gap)
        for g, red in zip(got, ("max", "sum", "count")):
            exp = O.spell_length_statistics(x, thr, 3, win_reducer, op, red, poff, min_gap=min_gap)
            np.testing.assert_array_equal(g.values, exp, err_msg=f"{win_reducer} {op} {red} {freq} {min_gap}")


def test_indicator_indexers_on_dataarrays_on_device(cuda, monkeypatch):
    """atmos.<index>(DataArray, **indexer): the masked series runs as a device Field, the result is re-labelled
    as a DataArray (tests/mini_xarray.py stands in for xarray, absent from the image)."""
    import mini_xarray as mx
    from test_xarray_boundary import _indexer_scenario
    mx.install(monkeypatch)
    _indexer_scenario()
