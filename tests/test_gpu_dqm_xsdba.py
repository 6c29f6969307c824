"""DQM parity pin against the real xsdba (`xsdba.DetrendedQuantileMapping`).  Where xsdba does not import this module
SKIPS (it does not pass); DESIGN.md says "parity unpinned" until it runs on a machine where it does."""
import numpy as np
import pytest

xsdba = pytest.importorskip("xsdba")
xr = pytest.importorskip("xarray")

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind", ["+", "*"])
def test_dqm_matches_xsdba(cuda, kind):
    from xclim_b200 import sdba
    rng = np.random.default_rng(9)
    T, shape = 365 * 10, (2, 3)
    time = xr.date_range("1981-01-01", periods=T, freq="D", calendar="noleap", use_cftime=True)
    mk = lambda a, u: xr.DataArray(a.astype(np.float32), dims=("time", "lat", "lon"), coords={"time": time},  # noqa: E731
                                   attrs={"units": u})
    base = 285.0 if kind == "+" else 5.0
    ref = base + np.abs(3 * rng.standard_normal((T,) + shape))
    hist = base * 1.02 + np.abs(3.5 * rng.standard_normal((T,) + shape))
    sim = base * 1.03 + np.abs(3.5 * rng.standard_normal((T,) + shape)) + np.linspace(0, 1, T)[:, None, None]
    u = "K" if kind == "+" else "mm/d"
    print("xsdba version", getattr(xsdba, "__version__", "?"))
    theirs = xsdba.DetrendedQuantileMapping.train(mk(ref, u), mk(hist, u), nquantiles=20, kind=kind, group="time")
    ours = sdba.DetrendedQuantileMapping.train(mk(ref, u), mk(hist, u), nquantiles=20, kind=kind, group="time")
    for interp in ("linear", "nearest"):
        for detrend in (0, 1, 2):
            b = theirs.adjust(mk(sim, u), interp=interp, extrapolation="constant", detrend=detrend)
            a = ours.adjust(mk(sim, u), interp=interp, extrapolation="constant", detrend=detrend)
            np.testing.assert_allclose(a.values, b.transpose("time", "lat", "lon").values, rtol=1e-5)
