"""GPU parity: rolling+resample, rolling-window spells, empirical quantile mapping."""
import numpy as np
import pytest

from oracle import xclim_oracle as O
from xb_helpers import make_field

pytestmark = pytest.mark.gpu


def _pr(rng, T, shape, nan_frac=0.01):
    x = rng.gamma(0.4, 6.0, size=(T,) + shape).astype(np.float32)
    x[rng.random(x.shape) < 0.45] = 0.0
    x = (np.round(x * 4) / 4).astype(np.float32)
    x[rng.random(x.shape) < nan_frac] = np.nan
    return x


@pytest.mark.parametrize("window,center,wop,op", [(3, False, "sum", "max"), (5, True, "mean", "max"),
                                                  (14, False, "mean", "min"), (7, True, "max", "mean"),
                                                  (2, False, "min", "sum"), (31, True, "sum", "std"),
                                                  (1, False, "sum", "max")])
@pytest.mark.parametrize("shape", [(5, 6), (4, 6)])   # 30 cells: lane-per-cell kernel; 24: streaming 4-cell kernel
def test_rolling_resample(cuda, window, center, wop, op, shape):
    from xclim_b200 import generic
    rng = np.random.default_rng(41)
    x = _pr(rng, 800, shape)
    da = make_field(x, "2000-01-01", units="mm/d")
    for freq in ("YS", "MS"):
        got = generic.select_rolling_resample_op(da, op, window, window_center=center, window_op=wop, freq=freq)
        exp = O.select_rolling_resample_op(x.astype(np.float64), op, window, da.time.period_offsets(freq),
                                           window_center=center, window_op=wop)
        np.testing.assert_allclose(got.values, exp, rtol=1e-5, equal_nan=True)  # float reductions: 1e-5


def test_rolling_reference_known_answers(cuda):
    """tests/test_generic.py:35-67 (values) and max_n_day_precipitation_amount."""
    from xclim_b200 import generic, indices
    q = make_field(np.arange(1, 366 + 365 + 365 + 1, dtype=np.float32), "2000-01-01", units="m3 s-1")
    o = generic.select_rolling_resample_op(q, "max", window=14, window_center=False, window_op="mean")
    np.testing.assert_array_equal(o.values, [np.mean(np.arange(353, 367)), np.mean(np.arange(353 + 365, 367 + 365)),
                                             np.mean(np.arange(353 + 730, 367 + 730))])
    assert o.attrs["units"] == "m3 s-1"
    o = generic.select_rolling_resample_op(q, "max", window=3, window_center=True, window_op="sum", freq="MS")
    np.testing.assert_array_equal(o.values[:2], [30 + 31 + 32, 59 + 60 + 61])
    pr = np.zeros(365, np.float32); pr[10:13] = [5, 7, 2]
    out = indices.max_n_day_precipitation_amount(make_field(pr, "2001-01-01", units="mm/d"), window=2)
    assert out.values[0] == 12 and out.attrs["units"] == "mm"


@pytest.mark.parametrize("window,winred,op,thr", [(3, "min", ">=", 1.0), (3, "max", "<", 1.0), (5, "sum", "<", 3.0),
                                                  (2, "mean", ">=", 2.0), (7, "sum", ">=", 20.0),
                                                  (30, "sum", "<", 40.0), (4, "max", ">", 6.0)])
@pytest.mark.parametrize("before", [True, False])
@pytest.mark.parametrize("shape", [(4, 5), (3, 5)])   # 20 cells: streaming 4-cell kernel; 15: lane-per-cell
def test_spell_length_statistics_windows(cuda, window, winred, op, thr, before, shape):
    from xclim_b200 import generic
    rng = np.random.default_rng(42)
    x = _pr(rng, 365 * 2 + 60, shape)
    da = make_field(x, "2001-01-01", units="mm/d")
    for freq in ("YS", "MS"):
        poff = da.time.period_offsets(freq)
        for red in ("max", "sum", "count"):
            got = generic.spell_length_statistics(da, thr, window, winred, op, red, freq, resample_before_rl=before)
            exp = O.spell_length_statistics(x, thr, window, winred, op, red, poff, resample_before_rl=before)
            np.testing.assert_array_equal(got.values, exp, err_msg=f"{window} {winred} {op} {red} {freq} {before}")


def test_spell_mask_reference_truth_tables(cuda):
    """tests/test_generic.py:702-713 through the statistics (total spell length == number of True)."""
    from xclim_b200 import generic
    data = make_field(np.array([0, 1, 2, 3, 2, 1, 0, 0], np.float32), "2001-01-01", units="")
    for window, red, op, thr, mask in [(3, "min", ">=", 2, [0, 0, 1, 1, 1, 0, 0, 0]),
                                       (3, "max", ">=", 2, [1, 1, 1, 1, 1, 1, 1, 0]),
                                       (2, "mean", ">=", 2, [0, 0, 1, 1, 1, 0, 0, 0])]:
        out = generic.spell_length_statistics(data, thr, window, red, op, "sum", "YS")
        assert out.values[0] == sum(mask)
        np.testing.assert_array_equal(O.spell_mask(data.values, window, red, op, thr), np.array(mask, bool))


@pytest.mark.parametrize("pr,thresh1,thresh2,window,outs", [
    ([1.01] * 6 + [0.01] * 3 + [0.51] * 2 + [0.75] * 2 + [0.51] + [0.01] * 3 + [1.01] * 3, 3, 3, 7, (1, 12, 20, 12, 20)),
    ([0.01] * 6 + [1.01] * 3 + [0.51] * 2 + [0.75] * 2 + [0.51] + [0.01] * 3 + [0.01] * 3, 3, 3, 7, (2, 18, 20, 10, 20)),
    ([3.01] * 358 + [0.99] * 14 + [3.01] * 358, 1, 14, 14, (0, 7, 7, 7, 7)),
])
def test_dry_spell_reference_known_answers(cuda, pr, thresh1, thresh2, window, outs):
    """tests/test_indices.py:4069-4112 (rtol=1e-1 as in the reference)."""
    from xclim_b200 import indices
    da = make_field(np.array(pr, np.float32), "1981-01-01", units="mm/day")
    ev, tds, tdm, mds, mdm = outs
    np.testing.assert_allclose(indices.dry_spell_frequency(da, thresh=f"{thresh1} mm", window=window).values[0], ev,
                               rtol=1e-1)
    np.testing.assert_allclose(indices.dry_spell_total_length(da, thresh=f"{thresh2} mm", window=window,
                                                              op="sum").values[0], tds, rtol=1e-1)
    np.testing.assert_allclose(indices.dry_spell_total_length(da, thresh=f"{thresh1} mm", window=window,
                                                              op="max").values[0], tdm, rtol=1e-1)
    np.testing.assert_allclose(indices.dry_spell_max_length(da, thresh=f"{thresh2} mm", window=window,
                                                            op="sum").values[0], mds, rtol=1e-1)
    np.testing.assert_allclose(indices.dry_spell_max_length(da, thresh=f"{thresh1} mm", window=window,
                                                            op="max").values[0], mdm, rtol=1e-1)


@pytest.mark.parametrize("kind,interp", [("+", "linear"), ("+", "nearest"), ("*", "linear")])
def test_eqm_train_adjust(cuda, kind, interp):
    """EQM vs the numpy restatement (PARITY UNPINNED against xsdba itself): train and nearest adjust bit for bit;
    linear adjust within 1e-5 relative (the oracle interpolates in float64, the kernel in float32)."""
    from xclim_b200 import sdba
    rng = np.random.default_rng(43)
    T, shape = 2000, (3, 4)
    ref = (285 + 6 * rng.standard_normal((T,) + shape)).astype(np.float32)
    hist = (286.5 + 7 * rng.standard_normal((T,) + shape)).astype(np.float32)
    sim = (288.5 + 7 * rng.standard_normal((T,) + shape)).astype(np.float32)
    hist[rng.random(hist.shape) < 0.01] = np.nan
    sim[rng.random(sim.shape) < 0.01] = np.nan
    ref[:, 0, 0] = np.nan   # untrainable cell -> NaN output
    f = lambda a: make_field(a, "1981-01-01", calendar="noleap", units="K")
    eqm = sdba.EmpiricalQuantileMapping.train(f(ref), f(hist), nquantiles=20, kind=kind, group="time")
    af_o, hq_o = O.eqm_train(ref, hist, 20, kind)
    ds = eqm.ds
    np.testing.assert_array_equal(ds["hist_q"].values, hq_o)
    np.testing.assert_array_equal(ds["af"].values, af_o)
    scen = eqm.adjust(f(sim), interp=interp, extrapolation="constant")
    exp = O.eqm_adjust(sim, ds["af"].values, ds["hist_q"].values, kind, interp)
    assert scen.values.dtype == np.float32 and scen.values.shape == sim.shape
    if interp == "nearest":
        np.testing.assert_array_equal(scen.values, exp)
    else:
        np.testing.assert_allclose(scen.values, exp, rtol=1e-5, equal_nan=True)
    # property (tests/test_xsdba.py:112-155 spirit): adjusting hist itself maps its quantiles onto ref's
    if kind == "+" and interp == "linear":
        back = eqm.adjust(f(hist), interp="linear").values[:, 1, 1]
        q = np.nanquantile(back, [0.25, 0.5, 0.75])
        np.testing.assert_allclose(q, np.nanquantile(ref[:, 1, 1], [0.25, 0.5, 0.75]), atol=0.15)


def test_eqm_train_heavy_ties_and_degenerate(cuda):
    """Multi-select edge cases: a heavy bin of exact ties (dry days), heavy bins that are NOT constant
    (forces the sort fallback), constant series, tiny series, all-NaN."""
    import torch
    from xclim_b200 import device
    rng = np.random.default_rng(44)
    T, C = 3000, 8
    ref = rng.gamma(0.5, 5.0, size=(T, C)).astype(np.float32)
    hist = rng.gamma(0.6, 4.0, size=(T, C)).astype(np.float32)
    ref[rng.random(ref.shape) < 0.5] = 0.0          # half the days are exactly 0
    hist[rng.random(hist.shape) < 0.6] = 0.0
    ref[:, 1] = 3.25                                # constant series
    hist[:, 2] = np.where(rng.random(T) < 0.5, 1.0, 1.0 + 1e-6).astype(np.float32)   # two values in one bin
    hist[:2, 2] = [0.0, 1000.0]                     # ... inside a wide range -> heavy, non-constant bin
    ref[:, 3] = np.nan                              # all NaN
    hist[5:, 4] = np.nan                            # only five valid values
    af, hq = device.eqm_train(torch.from_numpy(ref).cuda(), torch.from_numpy(hist).cuda(), 20, 0)
    af_o, hq_o = O.eqm_train(ref, hist, 20, "+")
    np.testing.assert_array_equal(hq.cpu().numpy(), hq_o)
    np.testing.assert_array_equal(af.cpu().numpy(), af_o)


@pytest.mark.parametrize("min_gap", [2, 3, 5])
@pytest.mark.parametrize("op,thr", [("<", 1.0), (">=", 4.0)])
def test_spell_length_statistics_min_gap(cuda, min_gap, op, thr):
    """generic.spell_mask(min_gap > 1) = runs_with_holes (indices/run_length.py:844-888): short gaps are
    bridged, a short gap running into the end of the series too, a gap that starts the series is not."""
    from xclim_b200 import generic
    rng = np.random.default_rng(44)
    x = _pr(rng, 365 * 2 + 40, (3, 7))
    x[:3, 0, 0] = 0.0; x[3, 0, 0] = 9.0           # series starts inside a short gap
    x[-2:, 0, 1] = 0.0; x[-3, 0, 1] = 9.0          # series ends inside a short gap
    da = make_field(x, "2001-01-01", units="mm/d")
    for freq in ("YS", "MS"):
        poff = da.time.period_offsets(freq)
        for red in ("max", "sum", "count", "mean"):
            got = generic.spell_length_statistics(da, thr, 1, None, op, red, freq, min_gap=min_gap)
            exp = O.spell_length_statistics(x, thr, 1, None, op, red, poff, min_gap=min_gap)
            np.testing.assert_array_equal(got.values, exp, err_msg=f"{min_gap} {op} {red} {freq}")
    with pytest.raises(NotImplementedError):
        generic.spell_length_statistics(da, thr, 3, "sum", op, "max", "YS", min_gap=2, resample_before_rl=False)


def test_eqm_train_group_kernels_match_one_cell_kernel(cuda, monkeypatch):
    """The cell-group multi-select (32 cells per CTA on the first 64 cells; 16 cells per CTA on all 80, which is not a
    multiple of 32, and on the first 48) bit for bit against the one-cell-per-CTA kernel and the oracle; the groups
    hold an all-NaN cell, a constant cell, a cell that needs the redo list (heavy non-constant bin), one whose range
    is subnormal (scale overflow -> redo), a precipitation-like cell with a heavy constant bin, cells full of ties."""
    import torch
    from xclim_b200 import device
    rng = np.random.default_rng(45)
    T, C = 10950, 80
    ref = (285 + 6 * rng.standard_normal((T, C))).astype(np.float32)
    hist = (286.5 + 7 * rng.standard_normal((T, C))).astype(np.float32)
    hist[rng.random(hist.shape) < 0.01] = np.nan
    ref[:, 3] = np.nan
    hist[:, 9] = 280.0
    hist[:, 17] = np.where(rng.random(T) < 0.5, 1.0, 1.0 + 1e-6).astype(np.float32)
    hist[:2, 17] = [0.0, 1000.0]                     # heavy, non-constant bin -> redo list
    pr = rng.gamma(0.5, 5.0, size=(T,)).astype(np.float32)
    pr[rng.random(T) < 0.5] = 0.0
    ref[:, 20] = pr                                  # heavy constant bin (dry days)
    ref[:, 40] = (rng.integers(0, 7, T) * np.float32(1e-42)).astype(np.float32)   # subnormal range
    hist[:, 41] = np.round(hist[:, 41])              # many ties
    ref[:, 50] = rng.integers(0, 3, T).astype(np.float32)                          # three values only
    rd, hd = torch.from_numpy(ref).cuda(), torch.from_numpy(hist).cuda()
    r64, h64 = rd[:, :64].contiguous(), hd[:, :64].contiguous()
    monkeypatch.delenv("XCLIM_B200_EQM_V1", raising=False)
    af, hq = device.eqm_train(rd, hd, 20, 0)                 # C % 32 != 0 -> 16 cells per CTA
    others = [device.eqm_train(r64, h64, 20, 0),             # 32 cells per CTA
              device.eqm_train(rd[:, :48].contiguous(), hd[:, :48].contiguous(), 20, 0)]   # 16 cells per CTA
    monkeypatch.setenv("XCLIM_B200_EQM_V1", "1")
    others.append(device.eqm_train(rd, hd, 20, 0))           # one cell per CTA
    torch.cuda.synchronize()
    for a_, h_ in others:
        n = a_.shape[1]
        assert torch.equal(torch.nan_to_num(af[:, :n], nan=-7.0), torch.nan_to_num(a_, nan=-7.0))
        assert torch.equal(torch.nan_to_num(hq[:, :n], nan=-7.0), torch.nan_to_num(h_, nan=-7.0))
    monkeypatch.delenv("XCLIM_B200_EQM_V1", raising=False)
    for nq in (1, 7, 50):                                    # 50 quantiles: the targets of 32 cells do not fit -> 16
        a_g, h_g = device.eqm_train(r64, h64, nq, 1)
        monkeypatch.setenv("XCLIM_B200_EQM_V1", "1")
        a_1, h_1 = device.eqm_train(r64, h64, nq, 1)
        monkeypatch.delenv("XCLIM_B200_EQM_V1", raising=False)
        assert torch.equal(torch.nan_to_num(a_g, nan=-7.0), torch.nan_to_num(a_1, nan=-7.0)), nq
        assert torch.equal(torch.nan_to_num(h_g, nan=-7.0), torch.nan_to_num(h_1, nan=-7.0)), nq
    af_o, hq_o = O.eqm_train(ref, hist, 20, "+")
    np.testing.assert_array_equal(hq.cpu().numpy(), hq_o)
    np.testing.assert_array_equal(af.cpu().numpy(), af_o)
