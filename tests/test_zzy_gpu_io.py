"""GPU: file-backed lazy sources (NetCDF-3, zarr v2) through the slab streamer (SURVEY.md 8f.3).  The host logic
also runs in tests/test_io_formats.py on CPU stand-ins."""
import numpy as np
import pytest

from xb_helpers import make_field

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind", ["netcdf3", "zarr"])
def test_file_in_file_out_through_the_streamer(cuda, tmp_path, kind):
    import xclim_b200
    from xclim_b200 import atmos, calendar as xcal, indices, io
    rng = np.random.default_rng(74)
    T, shape = 365 * 4, (11, 16)
    pr = rng.gamma(0.4, 6.0, size=(T,) + shape).astype(np.float32)
    pr[rng.random(pr.shape) < 0.5] = 0
    pr[rng.random(pr.shape) < 0.002] = np.nan
    tas = (285 + 10 * np.sin(2 * np.pi * (np.arange(T) % 365 - 110) / 365)[:, None, None]
           + 3 * rng.standard_normal((T,) + shape)).astype(np.float32)
    dims = ("time", "lat", "lon")
    f_pr = make_field(pr, "1981-01-01", calendar="noleap", units="mm/d", dims=dims)
    f_tas = make_field(tas, "1981-01-01", calendar="noleap", units="K", dims=dims)
    if kind == "netcdf3":
        l_pr = io.open_field(io.save_netcdf3(str(tmp_path / "pr.nc"), f_pr, name="pr"))
        l_tas = io.open_field(io.save_netcdf3(str(tmp_path / "tas.nc"), f_tas, name="tas"))
    else:
        l_pr = io.open_field(io.save_zarr(str(tmp_path / "pr.zarr"), f_pr, name="pr", chunks=(365, 4, 16)))
        l_tas = io.open_field(io.save_zarr(str(tmp_path / "tas.zarr"), f_tas, name="tas", chunks=(730, 3, 8),
                                           compressor=None))
    assert isinstance(l_pr.values, io.LazyGrid) and l_pr.time.calendar == "noleap"
    ref_cdd = atmos.maximum_consecutive_dry_days(f_pr).values
    ref_wet = indices.wetdays(f_pr).values
    per_ref = xcal.percentile_doy(f_tas, window=5, per=90.0)
    ref_tx = indices.tx90p(f_tas, xcal.select_percentile(per_ref, 90.0)).values
    row = T * shape[1] * 4
    with xclim_b200.set_options(stream_min_bytes=0, stream_slab_bytes=2 * row):
        cdd = atmos.maximum_consecutive_dry_days(l_pr)
        wet = indices.wetdays(l_pr)
        per = xcal.percentile_doy(l_tas, window=5, per=90.0)
        tx = indices.tx90p(l_tas, xcal.select_percentile(per, 90.0))
    np.testing.assert_array_equal(cdd.values, ref_cdd)
    np.testing.assert_array_equal(wet.values, ref_wet)
    np.testing.assert_array_equal(per.values, per_ref.values)
    np.testing.assert_array_equal(tx.values, ref_tx)
    # small inputs: the lazy source is materialised once and takes the one-piece path
    np.testing.assert_array_equal(atmos.maximum_consecutive_dry_days(l_pr).values, ref_cdd)
    out = io.save_zarr(str(tmp_path / "cdd.zarr"), cdd, name="cdd", calendar="noleap")
    back = io.open_field(out, "cdd")
    np.testing.assert_array_equal(np.asarray(back.values), ref_cdd)
    assert back.attrs["units"] == "days"
